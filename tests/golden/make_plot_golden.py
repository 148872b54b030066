#!/usr/bin/env python3
"""Golden fixtures for `haphic plot`, made by the REFERENCE's own code:

    python tests/golden/make_plot_golden.py

Imports scripts/HapHiC_plot.py of the reference unmodified, with PYTHONHASHSEED=0 and stand-ins for pysam (only
set_verbosity is reached on the .pairs path), portion (closed intervals: &, in, lower / upper, hash / eq) and matplotlib
(never drawn: the draw functions are replaced by no-ops).  Writes tests/golden/plot_<case>.npz with the AGP and .pairs text,
the layout the golden positions resolve to, the symmetrised matrix, normalize_matrix's outputs (KR / log10) and vmax for
KR / log10 / none, the log lines, the contents of main()'s contact_matrix.pkl, and (plot_bnewt.npz) bnewt's x with its
outer and inner step counts for every block and whole matrix of the cases and a random one."""

import logging
import os
import pickle
import sys
import tempfile
import types

if os.environ.get("PYTHONHASHSEED") != "0":
    os.environ["PYTHONHASHSEED"] = "0"
    os.execv(sys.executable, [sys.executable] + sys.argv)

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
sys.path.insert(0, HERE)

import numpy as np

from make_golden import REF  # the reference's scripts directory

U = 100_000          # the cases use --bin_size 100 (kb)


class Closed:
    """A closed integer interval as HapHiC_plot.py uses portion.closed."""

    def __init__(self, lo, hi):
        self.lower, self.upper = lo, hi

    def __and__(self, other):
        return Closed(max(self.lower, other.lower), min(self.upper, other.upper))

    def __contains__(self, v):
        return self.lower <= v <= self.upper

    def __eq__(self, other):
        return (self.lower, self.upper) == (other.lower, other.upper)

    def __hash__(self):
        return hash((self.lower, self.upper))


def import_reference():
    pysam = types.ModuleType("pysam")
    pysam.set_verbosity = lambda *_a, **_k: 0
    portion = types.ModuleType("portion")
    portion.closed = Closed
    mpl = types.ModuleType("matplotlib")
    mpl.use = lambda *_a, **_k: None
    mpl.pyplot = types.ModuleType("matplotlib.pyplot")
    mpl.colors = types.ModuleType("matplotlib.colors")
    for name, mod in (("pysam", pysam), ("portion", portion), ("matplotlib", mpl), ("matplotlib.pyplot", mpl.pyplot),
                      ("matplotlib.colors", mpl.colors)):
        sys.modules[name] = mod
    sys.path.insert(0, REF)
    import HapHiC_plot as ref
    return ref


# ---- inputs -------------------------------------------------------------------------------------------------------

def layout_pieces():
    """Scaffolds as lists of W pieces (contig, raw_start, raw_end, ori) and U gaps (None, length)."""
    S1 = [("A", 1, 25 * U, "+"), (None, 1000), ("B", 1, 18 * U, "-"), (None, 500), ("C", 1, 10 * U, "+")]
    # C's second piece starts in the middle of an aln bin; the scaffold ends on an exact multiple of the bin size
    S2 = [("D", 1, 30 * U, "-"), (None, U), ("C", 20 * U + 50001, 30 * U, "+")]
    s2_len = 30 * U + U + (10 * U - 50000)
    S2.append(("E", 1, 50 * U - s2_len, "-"))
    S3 = [("F", 1, 6 * U, "+")]                       # 0.6 Mb: below --min_len 1
    S4 = [("G", 1, 12 * U, "-"), (None, 100), ("H", 1, 15 * U, "+")]
    return [("S1", S1), ("S2", S2), ("S3", S3), ("S4", S4)]


LENGTHS = {"A": 25 * U, "B": 18 * U, "C": 30 * U, "D": 30 * U, "E": 9 * U + 50000, "F": 6 * U, "G": 12 * U, "H": 15 * U,
           "X": 5 * U}


def agp_text():
    out = []
    for g, pieces in layout_pieces():
        pos, part = 1, 1
        for p in pieces:
            if p[0] is None:
                out.append("{}\t{}\t{}\t{}\tU\t{}\tscaffold\tyes\tproximity_ligation".format(g, pos, pos + p[1] - 1, part, p[1]))
                pos += p[1]
            else:
                c, rs, re_, ori = p
                n = re_ - rs + 1
                out.append("{}\t{}\t{}\t{}\tW\t{}\t{}\t{}\t{}".format(g, pos, pos + n - 1, part, c, rs, re_, ori))
                pos += n
            part += 1
    return "# AGP\n" + "\n".join(out) + "\n"


def special_positions():
    """(contig, 1-based position) at 1, bin_size, bin_size + 1 and every piece end of every placed contig."""
    pts = []
    for _g, pieces in layout_pieces():
        for p in pieces:
            if p[0] is not None:
                c, rs, re_, _o = p
                pts += [(c, rs), (c, re_), (c, rs + 1), (c, re_ - 1)]
    for c in LENGTHS:
        if c != "X":
            pts += [(c, 1), (c, U), (c, U + 1)]
    pts.append(("C", 20 * U + 10))            # listed aln bin, in no range: skip
    return pts


def make_pairs(seed, n, error_case=False):
    rng = np.random.default_rng(seed)
    names = [c for c in LENGTHS if c != "X"]
    placed = {"A": [(1, 25 * U)], "B": [(1, 18 * U)], "C": [(1, 10 * U), (20 * U + 50001, 30 * U)], "D": [(1, 30 * U)],
              "E": [(1, LENGTHS["E"])], "F": [(1, 6 * U)], "G": [(1, 12 * U)], "H": [(1, 15 * U)]}

    def draw_pos(c):
        lo, hi = placed[c][rng.integers(len(placed[c]))]
        return int(rng.integers(lo, hi + 1))

    rows = []
    for _ in range(n):
        a = names[rng.integers(len(names))]
        pa = draw_pos(a)
        if rng.random() < 0.6:
            b = a
            pb = min(max(1, pa + int(rng.normal(0, 3 * U))), LENGTHS[a])
            if not any(lo <= pb <= hi for lo, hi in placed[a]):
                pb = pa
        else:
            b = names[rng.integers(len(names))]
            pb = draw_pos(b)
        rows.append((a, pa, b, pb))
    sp = special_positions()
    for k, (c, p) in enumerate(sp):
        rows.insert(int(rng.integers(len(rows))), (c, p, *sp[(k * 7 + 3) % len(sp)]))
        rows.insert(int(rng.integers(len(rows))), (sp[(k * 5 + 1) % len(sp)][0], sp[(k * 5 + 1) % len(sp)][1], c, p))
    rows.insert(10, ("X", 5, "A", 7))             # a name missing from the AGP
    rows.insert(20, ("A", 9, "X", 5))
    if error_case:
        # first end skips (C in a listed bin but no range), second unplaceable: no error; then the first real error
        rows.insert(30, ("C", 20 * U + 10, "C", 15 * U))
        rows.insert(40, ("A", 100, "C", 15 * U + 7))
        rows.insert(50, ("C", 12 * U, "A", 100))
    return rows


def pairs_text(rows):
    return "## pairs format v1.0\n#columns: readID chr1 pos1 chr2 pos2 strand1 strand2\n" + "".join(
        "r{}\t{}\t{}\t{}\t{}\t+\t-\n".format(i, a, pa, b, pb) for i, (a, pa, b, pb) in enumerate(rows))


# ---- cases --------------------------------------------------------------------------------------------------------

CASES = [
    ("main", dict(bin_size=100, min_len=1, specified_scaffolds=None), 1901, 20000, False),
    ("specified", dict(bin_size=100, min_len=1, specified_scaffolds="S4,S3,S1"), 1902, 20000, False),
    ("allkept", dict(bin_size=100, min_len=0, specified_scaffolds=None), 1903, 20000, False),
    ("error", dict(bin_size=100, min_len=1, specified_scaffolds=None), 1904, 2000, True),
]


class LogCapture(logging.Handler):
    def __init__(self):
        super().__init__()
        self.lines = []

    def emit(self, record):
        self.lines.append(record.getMessage())


def run_main(ref, agp, pairs, argv, workdir):
    """The reference's main() with the draw functions as no-ops; returns the pickle's contents and the log lines."""
    cap = LogCapture()
    ref.logger.addHandler(cap)
    ref.draw_heatmap = lambda *a, **k: None
    ref.draw_separate_heatmaps = lambda *a, **k: None
    old_argv, old_cwd = sys.argv, os.getcwd()
    sys.argv = ["HapHiC_plot.py", agp, pairs] + argv
    os.chdir(workdir)
    try:
        ref.main()
        with open("contact_matrix.pkl", "rb") as f:
            mat, args, md5 = pickle.load(f)
    finally:
        sys.argv = old_argv
        os.chdir(old_cwd)
        ref.logger.removeHandler(cap)
        for h in list(ref.logger.handlers):
            if isinstance(h, logging.FileHandler):
                ref.logger.removeHandler(h)
                h.close()
    return mat, args, md5, cap.lines


def argv_of(kw, extra=()):
    out = ["--bin_size", str(kw["bin_size"]), "--min_len", str(kw["min_len"])]
    if kw["specified_scaffolds"]:
        out += ["--specified_scaffolds", kw["specified_scaffolds"]]
    return out + list(extra)


class CountingMatrix(np.ndarray):
    """Counts A @ v calls, so that bnewt's inner steps can be recovered: calls = 1 + sum over outer steps (k + 1)."""
    calls = 0

    def __matmul__(self, other):
        CountingMatrix.calls += 1
        return np.asarray(self) @ other


def bnewt_counts(ref, A):
    CountingMatrix.calls = 0
    x, res = ref.bnewt(A.view(CountingMatrix), fl=1)
    outer = len(res)
    return np.asarray(x), outer, CountingMatrix.calls - 1 - outer


def main():
    ref = import_reference()
    ref.logger.setLevel(logging.INFO)
    tmp = tempfile.mkdtemp()
    agp = os.path.join(tmp, "asm.agp")
    with open(agp, "w") as f:
        f.write(agp_text())
    bnewt_mats = []
    for tag, kw, seed, n, err in CASES:
        rows = make_pairs(seed, n, err)
        pairs = os.path.join(tmp, "{}.pairs".format(tag))
        with open(pairs, "w") as f:
            f.write(pairs_text(rows))
        bs = kw["bin_size"] * 1000
        ctg_dict, ctg_aln_dict, group_size_dict, frag_set, group_frag_dict = ref.parse_agp(agp, bs)
        cm0, g2t, group_list, ctg_set = ref.generate_contact_matrix(group_size_dict, set(frag_set), group_frag_dict, bs,
                                                                    kw["min_len"], kw["specified_scaffolds"])
        # how the golden positions resolve (every special position and both ends of the first 2000 records): total bin,
        # -1 skip, -2 the reference raises.  The device tests check every record through the matrix.
        probes = sorted({(c, p) for r in rows[:2000] for (c, p) in ((r[0], r[1]), (r[2], r[3]))
                         if c in ctg_set} | {(c, p) for c, p in special_positions() if c in ctg_set})
        res = []
        for c, p in probes:
            try:
                v = None
                for rng_ in ctg_aln_dict[c][(p - 1) // bs]:
                    gb = ctg_dict[c][rng_]
                    if p in rng_:
                        v = -1 if gb[0] not in group_list else g2t[gb]
                        break
                res.append(-1 if v is None else v)
            except KeyError:
                res.append(-2)
        out = dict(agp=np.array(agp_text()), pairs=np.array(pairs_text(rows)), bin_size=kw["bin_size"],
                   min_len=kw["min_len"], specified=np.array(kw["specified_scaffolds"] or ""),
                   probe_ctg=np.array([c for c, _ in probes]), probe_pos=np.array([p for _, p in probes], np.int64),
                   probe_bin=np.array(res, np.int64), group_list=np.array(group_list), nb=cm0.shape[0],
                   in_ctg_set=np.array(sorted(ctg_set)))
        if err:
            try:
                ref.parse_pairs(pairs, ctg_dict, ctg_aln_dict, bs, cm0, g2t, group_list, ctg_set)
                raise AssertionError("the error case did not raise")
            except Exception as e:
                out["error"] = np.array(str(e))
            np.savez_compressed(os.path.join(HERE, "plot_{}.npz".format(tag)), **out)
            print(tag, "error:", out["error"])
            continue
        for norm in ("KR", "log10", "none"):
            wd = tempfile.mkdtemp(dir=tmp)
            mat, args, md5, lines = run_main(ref, agp, pairs, argv_of(kw, ["--normalization", norm]), wd)
            if norm == "KR":
                out["matrix"] = mat
                out["pkl_args"] = np.array(repr(list(vars(args).items())))
                out["pkl_md5"] = np.array(md5)
            nm, vmax = ref.normalize_matrix(mat, group_list, group_size_dict, bs, norm, 4.0, -1)
            if norm != "none":              # the raw matrix itself
                out["norm_" + norm] = np.asarray(nm, np.float64)
            out["vmax_" + norm] = np.float64(vmax)
            out["log_" + norm] = np.array([ln for ln in lines if "vmax" in ln or "Normaliz" in ln])
        # bnewt on the whole matrix and on each block
        A = out["matrix"] + 0.00001
        start = 0
        for g in group_list:
            nbin = int(np.ceil(group_size_dict[g] / bs))
            bnewt_mats.append(("{}_{}".format(tag, g), A[start:start + nbin, start:start + nbin].copy()))
            start += nbin
        bnewt_mats.append(("{}_whole".format(tag), A.copy()))
        np.savez_compressed(os.path.join(HERE, "plot_{}.npz".format(tag)), **out)
        print(tag, "nb", cm0.shape[0], "vmax", [float(out["vmax_" + k]) for k in ("KR", "log10", "none")])
    rng = np.random.default_rng(7)
    R = rng.poisson(3.0, (40, 40)).astype(np.int64)
    bnewt_mats.append(("random40", (R + R.T) + 0.00001))
    bout = {}
    for name, A in bnewt_mats:
        x, outer, inner = bnewt_counts(ref, A)
        bout["A_" + name], bout["x_" + name] = A, x
        bout["steps_" + name] = np.array([outer, inner], np.int64)
        print("bnewt", name, A.shape[0], outer, inner)
    bout["names"] = np.array([name for name, _ in bnewt_mats])
    np.savez_compressed(os.path.join(HERE, "plot_bnewt.npz"), **bout)


if __name__ == "__main__":
    main()
