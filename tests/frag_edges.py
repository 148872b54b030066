"""The edges layout of fragment mode (contigs split into bins) and seeded record streams over it.  Shared by
tests/golden/make_golden.py (links_bins_edges.npz, made with the reference), tests/test_frag_oracle.py and
tests/test_gpu_links_frags.py.

With 10 kb bins: ctg1 has 13 bins (the last one 5 kb), ctg1A is exactly one bin long (not split), ctg1_x one bin + 1 bp
(a last bin of 1 bp), ctg1a exactly 3 bins, ctg2 2.5 bins; ctg10 and ctg3 are shorter than a bin.  Appending '_binK'
flips name orders, since '0' < 'A' < '_' < 'a': ctg1 < ctg10 but ctg10 < ctg1_bin1, and
ctg1A < ctg1_bin1 < ctg1_bin10 < ctg1_bin2 < ctg1_x_bin1 < ctg1a_bin1.  The contigs are not in name order."""

import numpy as np

BIN_KB = 10
LAYOUT = (("ctg2", 25000), ("ctg1", 125000), ("ctg10", 8000), ("ctg1A", 10000), ("ctg1_x", 10001), ("ctg3", 4000),
          ("ctg1a", 30000))
GHOST = "ghost_ctg"          # a contig missing from the FASTA: id len(LAYOUT) in the records

# single records whose outcome in parse_alignments is pinned one by one: (ctg, pos, ctg, pos), 0-based positions
SINGLE = (
    ("ctg1", -1, "ctg1", -1),              # both ends in the missing bin 0: skipped (1715)
    ("ctg1", 200000, "ctg1", 200500),      # both ends in the missing bin 21: skipped
    ("ctg1", -10000, "ctg1", -1),          # both in bin 0 (floor division, not truncation): skipped
    ("ctg1_x", 20000, "ctg1_x", 20001),    # both in the missing bin 3 of a 2-bin contig: skipped
    ("ctg1", -1, "ctg2", 5),               # missing bin x existing bin: KeyError (1723)
    ("ctg1", -1, "ctg1", 5),               # missing bin 0 x bin 1 of the same contig: KeyError
    ("ctg1", -10001, "ctg1", -5),          # bins -1 and 0: KeyError
    ("ctg1", 130000, "ctg2", 0),           # bin 14 of a 13-bin contig: KeyError
    ("ctg1a", 30000, "ctg1a", 29999),      # bin 4 of a 3-bin contig x its bin 3: KeyError
    ("ctg10", 3, "ctg1_x", 20001),         # bin 3 of a 2-bin contig x an unsplit one: KeyError
    ("ctg1", 125000, "ctg2", 5),           # past the contig's end but inside its last bin (13): counted
    ("ctg1", 129999, "ctg3", 5),           # the last position of bin 13: counted
    ("ctg1A", 50000, "ctg2", 5),           # past the end of an unsplit contig: no bins, counted
    ("ctg10", -1, "ctg3", 5),              # position -1 on unsplit contigs: counted
    ("ctg1_x", 10000, "ctg1_x", 10000),    # equal positions in the 1-bp last bin: skipped
    ("ctg1_x", 9999, "ctg1_x", 10000),     # the two bins of ctg1_x: counted
    (GHOST, 5, "ctg1", -1),                # a contig missing from the FASTA: skipped (1703) before any bin
    ("ctg3", 5, "ctg3", 7),                # intra-contig on an unsplit contig: skipped (1699)
)
SKIPPED, COUNTED, RAISES = 0, 1, 2


def names():
    return [n for n, _ in LAYOUT]


def lengths():
    return np.array([ln for _, ln in LAYOUT], np.int64)


def stream(n_rec, seed):
    """n_rec records (contig ids, 0-based positions) over LAYOUT: half of the ends at 0, bin_size - 1, bin_size, every
    k * bin_size - 1 and k * bin_size, or len - 1, the others uniform; intra-contig pairs on split contigs in one bin, in
    adjacent bins, in the first and last bins and at equal positions; inter-contig pairs split x split, split x unsplit
    and unsplit x unsplit, either end first; 1 % of the records name the missing contig.  No record names a bin that
    does not exist."""
    rng = np.random.default_rng(seed)
    bs = BIN_KB * 1000
    ln = lengths()
    n = len(ln)
    split, unsplit = np.nonzero(ln > bs)[0], np.nonzero(ln <= bs)[0]
    kind = rng.integers(0, 8, n_rec)
    a, b = rng.integers(0, n, n_rec), rng.integers(0, n, n_rec)
    for k, (sa, sb) in {0: (split, None), 1: (split, None), 2: (split, None), 3: (split, None), 4: (split, split),
                        5: (split, unsplit), 6: (unsplit, unsplit)}.items():
        m = kind == k
        a[m] = sa[rng.integers(0, len(sa), int(m.sum()))]
        b[m] = a[m] if sb is None else sb[rng.integers(0, len(sb), int(m.sum()))]
    pos = np.empty((n_rec, 2), np.int64)
    for c in range(n):
        edges = np.array(sorted({p for k in range(int(ln[c]) // bs + 2) for p in (k * bs - 1, k * bs) if 0 <= p < ln[c]}
                                | {int(ln[c]) - 1}), np.int64)
        for col, ends in ((0, a), (1, b)):
            m = ends == c
            cnt = int(m.sum())
            pos[m, col] = np.where(rng.random(cnt) < 0.5, edges[rng.integers(0, len(edges), cnt)], rng.integers(0, ln[c], cnt))
    # intra-contig layouts: 0 one bin, 1 adjacent bins across a bin edge, 2 first and last bin, 3 equal positions
    la = ln[a]
    bin_k = rng.integers(0, 1 << 30, n_rec) % np.maximum(-(-la // bs) - 1, 1)
    m = kind == 0
    lo, hi = bin_k[m] * bs, np.minimum((bin_k[m] + 1) * bs, la[m])
    pos[m, 0] = lo + rng.integers(0, 1 << 30, int(m.sum())) % (hi - lo)
    pos[m, 1] = lo + rng.integers(0, 1 << 30, int(m.sum())) % (hi - lo)
    m = kind == 1
    pos[m, 0] = (bin_k[m] + 1) * bs - 1 - rng.integers(0, 3, int(m.sum()))
    pos[m, 1] = np.minimum((bin_k[m] + 1) * bs + rng.integers(0, 3, int(m.sum())), la[m] - 1)
    m = kind == 2
    pos[m, 0] = rng.integers(0, 2, int(m.sum()))
    pos[m, 1] = la[m] - 1 - rng.integers(0, 2, int(m.sum()))
    m = kind == 3
    pos[m, 1] = pos[m, 0]
    flip = rng.random(n_rec) < 0.5
    rec = np.stack([np.where(flip, b, a), np.where(flip, pos[:, 1], pos[:, 0]),
                    np.where(flip, a, b), np.where(flip, pos[:, 0], pos[:, 1])], 1)
    ghost = rng.random(n_rec) < 0.01
    side = rng.integers(0, 2, n_rec)
    rec[ghost & (side == 0), 0] = n
    rec[ghost & (side == 1), 2] = n
    return rec.astype(np.int32)


def single_records():
    """SINGLE as int32 [S, 4] contig-id records (GHOST = id len(LAYOUT))."""
    ids = {nm: i for i, nm in enumerate(names() + [GHOST])}
    return np.array([[ids[a], pa, ids[b], pb] for a, pa, b, pb in SINGLE], np.int32)
