#!/usr/bin/env python3
"""Golden fixtures for `haphic cluster --ul` (ultra-long read contig paths), made by the REFERENCE's own code:

    python tests/golden/make_ul_golden.py

Imports scripts/HapHiC_cluster.py of the reference unmodified, the way make_gfa_golden.py does (same stubs,
PYTHONHASHSEED=0), with _pysam_ul.AlignmentFile standing in for pysam and a small closed-interval class for `portion`.
Writes
  * ul_parse.npz -- parse_ul_alignments' path_list on the adversarial UL BAM (synth.ul_adversarial) for several
    --min_ul_support values;
  * ul_<case>.npz -- whole runs: path_list, whitelist, output files, typed full_links.pkl / HT_links.pkl items and the
    log lines of the functions --ul touches."""

import json
import logging
import os
import pickle
import sys
import tempfile

if os.environ.get("PYTHONHASHSEED") != "0":
    os.environ["PYTHONHASHSEED"] = "0"
    os.execv(sys.executable, [sys.executable] + sys.argv)

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
sys.path.insert(0, HERE)

import numpy as np

import _portion
import _pysam_ul
from make_golden import import_reference, make_args
from make_gfa_golden import blob, sha, typed_items


class _Closed:
    """The closed integer intervals portion gives parse_ul_alignments: &, |, complement()[1], lower / upper, truth."""

    def __init__(self, atoms):
        self.atoms = [a for a in atoms if a[0] <= a[1]]

    lower = property(lambda self: self.atoms[0][0])
    upper = property(lambda self: self.atoms[-1][1])

    def __bool__(self):
        return bool(self.atoms)

    def __and__(self, other):
        (a, b), (c, d) = self.atoms[0], other.atoms[0]
        return _Closed([(max(a, c), min(b, d))])

    def __or__(self, other):
        return _Closed(sorted(self.atoms + other.atoms))

    def complement(self):
        # the gaps between the atoms as open intervals (lower, upper); [0] and [-1] are the unbounded ends
        inf = float("inf")
        return [_Closed([(-inf, self.atoms[0][0])])] + [_Open(self.atoms[k][1], self.atoms[k + 1][0])
                                                         for k in range(len(self.atoms) - 1)] + [None]


class _Open:
    def __init__(self, lower, upper):
        self.lower, self.upper = lower, upper


SWEEP = dict(min_inflation=1.4, max_inflation=2.2, inflation_step=0.4)
# (tag, nchr, n_contigs, mean_len, n_pairs, seed, ploidy, n_gfa, no_path, argkw)
RUN_CASES = [
    ("ctg", 4, 80, 50000, 100000, 1801, 1, 0, False, dict(Nx=100, bin_size=0, **SWEEP)),
    ("bins", 4, 40, 200000, 100000, 1802, 1, 0, False, dict(Nx=100, bin_size=120, flank=60, **SWEEP)),
    ("norm", 4, 80, 50000, 100000, 1803, 1, 0, False, dict(Nx=100, bin_size=0, normalize_by_nlinks=True, **SWEEP)),
    ("gfa_w05", 4, 80, 50000, 100000, 1804, 2, 2, False, dict(Nx=100, bin_size=0, phasing_weight=0.5, **SWEEP)),
    ("gfa_w1", 4, 80, 50000, 100000, 1804, 2, 2, False, dict(Nx=100, bin_size=0, **SWEEP)),
    ("allelic", 4, 80, 50000, 100000, 1805, 2, 0, False, dict(Nx=100, bin_size=0, remove_allelic_links=2, **SWEEP)),
    ("concentrated", 4, 80, 50000, 100000, 1806, 1, 0, False, dict(Nx=100, bin_size=0, remove_concentrated_links=True,
                                                                    **SWEEP)),
    ("quick_view", 4, 80, 50000, 100000, 1807, 1, 0, False, dict(quick_view=True)),
    ("no_path", 4, 80, 50000, 100000, 1809, 1, 0, True, dict(Nx=100, bin_size=0, **SWEEP)),
    # --ul with --correct_nrounds is dropped with a warning (2774-2776); correction itself uses portion
    ("correct", 4, 80, 50000, 100000, 1808, 1, 0, False, dict(Nx=100, bin_size=0, correct_nrounds=2, **SWEEP)),
]
LOGGED = ("parse_ul_alignments", "filter_fragments", "reduce_inter_hap_HiC_links", "recommend_inflation", "mcl", "run",
          "stat_fragments")


def run_case(ref, tag, nchr, n_contigs, mean_len, n_pairs, seed, ploidy, n_gfa, no_path, argkw):
    from haphic_b200 import synth
    out, rec = {}, {}
    orig = ref.parse_ul_alignments

    def parse_wrap(args):
        got = orig(args)
        rec["path_list"] = [list(p) for p in got]
        return got

    ref.parse_ul_alignments = parse_wrap
    ul_closed = ref.closed
    if argkw.get("correct_nrounds"):
        ref.closed, ref.empty = _portion.closed, _portion.empty
    with tempfile.TemporaryDirectory() as tmp:
        cwd = os.getcwd()
        os.chdir(tmp)
        try:
            gfa = synth.ul_case(nchr, n_contigs, mean_len, n_pairs, seed, tmp, ploidy=ploidy, n_gfa=n_gfa, no_path=no_path)
            args = make_args(fasta=os.path.join(tmp, "asm.fa"), alignments=os.path.join(tmp, "aln.pairs"), nchrs=nchr,
                             gfa=",".join(gfa) if gfa else None, ul=os.path.join(tmp, "ul.bam"), **argkw)
            ref.INTEL_MKL = True
            ref.dot_product_mkl = lambda a, b: a @ b
            ref.run(args, log_file="HapHiC_cluster.log")
            for h in list(ref.logger.handlers):
                if isinstance(h, logging.FileHandler):
                    h.close()
                    ref.logger.removeHandler(h)
            files, digests = {}, {}
            for root, _dirs, fnames in os.walk("."):
                for fn in fnames:
                    p = os.path.join(root, fn)[2:]
                    if p.startswith("inflation_") and p.endswith(".txt"):
                        with open(p) as f:
                            files[p] = f.read()
                    elif p.endswith((".pkl", ".clm", ".bed")):
                        with open(p, "rb") as f:
                            digests[p] = sha(f.read())
            with open("HapHiC_cluster.log") as f:
                log = f.read()
            lines = []
            for ln in log.splitlines():
                fn = ln.split("[", 1)[1].split("]", 1)[0] if "[" in ln else ""
                if fn in LOGGED:
                    lines.append("[{}] {}".format(fn, ln.split("] ", 1)[1]))
            out["log_lines"] = blob(lines)
            for name in ("full_links", "HT_links"):
                if os.path.exists(name + ".pkl"):
                    with open(name + ".pkl", "rb") as f:
                        out[name + "_items"] = blob(typed_items(pickle.load(f)))
            out["files_json"] = blob(files, sort_keys=True)
            out["digests_json"] = blob(digests, sort_keys=True)
            out["path_list"] = blob(rec.get("path_list", []))
            out["whitelist"] = blob(sorted(getattr(args, "whitelist", set())))
            out["argkw"] = blob(argkw, sort_keys=True)
            out["case"] = np.array([nchr, n_contigs, mean_len, n_pairs, seed, ploidy, n_gfa, no_path], dtype=np.int64)
        finally:
            os.chdir(cwd)
            ref.parse_ul_alignments = orig
            ref.closed = ul_closed
    np.savez_compressed(os.path.join(HERE, "ul_{}.npz".format(tag)), **out)
    print("ul_{}: {} files, {} log lines, {} paths".format(tag, len(files), len(lines), len(rec.get("path_list", []))))


def parse_cases(ref):
    """path_list of the adversarial BAM for several --min_ul_support values."""
    from haphic_b200 import hicio, synth
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        bam = os.path.join(tmp, "adv.bam")
        hicio.write_ul_bam(bam, *synth.ul_adversarial())
        for support in (1, 2, 3, 4):
            args = make_args(ul=bam, min_ul_support=support)
            out[str(support)] = [list(p) for p in ref.parse_ul_alignments(args)]
    np.savez_compressed(os.path.join(HERE, "ul_parse.npz"), paths_json=blob(out))
    print("ul_parse:", {k: len(v) for k, v in out.items()})


def main():
    sys.modules["pysam"] = _pysam_ul
    ref = import_reference()
    ref.pysam = _pysam_ul
    ref.closed = lambda lo, hi: _Closed([(lo, hi)])
    # networkx >= 3 returns the all-pairs shortest paths as a generator; the reference indexes them as the dict they were
    import networkx
    ref.shortest_path = lambda g: dict(networkx.shortest_path(g))
    only = set(sys.argv[1:])
    if not only or "parse" in only:
        parse_cases(ref)
    for case in RUN_CASES:
        if not only or case[0] in only:
            run_case(ref, *case)


if __name__ == "__main__":
    main()
