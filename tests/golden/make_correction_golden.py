#!/usr/bin/env python3
"""Golden fixtures for assembly correction (`--correct_nrounds`), made by the REFERENCE's own code:

    python tests/golden/make_correction_golden.py

Imports scripts/HapHiC_cluster.py of the reference unmodified, the way make_golden.py does, with a functional stand-in
for ``portion`` (tests/golden/_portion.py, written from portion's documented semantics) and records every round of
correct_assembly by wrapping detect_break_points at run time.  Writes tests/golden/correct_*.npz."""

import json
import os
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
from make_golden import import_reference, make_args

# every pairs case: (tag, nchr, n_contigs, mean_len, n_pairs, n_joins, span, seed, argkw); chimeras of three contigs for
# tags ending in g3.  The first half of the chimeras has planted spanning records (non-zero valleys), the second half
# zero-coverage gaps (synth.chimera_case).
# every whole run: (tag, nchr, n_contigs, mean_len, n_pairs, n_joins, span, seed, group, argkw)
PAIRS_CASES = [
    ("r1", 4, 120, 60000, 120000, 6, 40, 41, dict(correct_nrounds=1)),
    ("r2", 4, 120, 60000, 120000, 6, 40, 42, dict(correct_nrounds=2)),
    ("r4", 3, 90, 80000, 150000, 8, 30, 43, dict(correct_nrounds=4, correct_resolution=400)),
    ("r4g3", 4, 120, 60000, 200000, 6, 60, 44, dict(correct_nrounds=4)),
    # shallow non-zero valleys only (no gaps): breaks a fragment that does not start at 1 in round 2 of 4
    ("r4g3_nogap", 4, 120, 60000, 200000, 6, 60, 44, dict(correct_nrounds=4)),
]
RUN_CASES = [
    ("run_nobins", 4, 160, 50000, 150000, 6, 40, 51, 3, dict(correct_nrounds=2, Nx=100, bin_size=0, min_inflation=1.4,
                                                         max_inflation=2.2, inflation_step=0.4)),
    ("run_bins", 3, 60, 300000, 150000, 4, 40, 52, 2, dict(correct_nrounds=2, Nx=100, bin_size=120, flank=60, min_inflation=1.4,
                                                        max_inflation=2.2, inflation_step=0.4)),
    ("run_nobreak", 4, 160, 50000, 150000, 0, 0, 53, 2, dict(correct_nrounds=2, Nx=100, bin_size=0, min_inflation=1.4,
                                                         max_inflation=2.2, inflation_step=0.4)),
]

# hand-made coverage arrays for detect_break_points: (name, fragment length, coverage).  The lengths are those of a contig
# with exactly len(coverage) bins at resolution 500, (n - 1) * 500 + 250, so the same arrays can be built on the device.
FUNCTION_CASES = [
    ("median0", 3250, [0, 0, 0, 5, 5, 0, 0]),
    ("one_run", 7250, [5] * 12 + [0] * 3),
    ("small_runs", 13250, [9] * 3 + [0] + [9] * 3 + [1] * 20),
    ("one_large", 26250, [9] * 20 + [0] + [9] * 2 + [8] * 30),
    ("zero_valley", 14250, [9] * 12 + [3, 0, 2, 0] + [9] * 12 + [9]),
    ("two_zero_valleys", 19250, [9] * 12 + [0] + [9] * 12 + [1, 0] + [9] * 12),
    ("mixed_valleys", 19750, [9] * 12 + [2, 1] + [9] * 12 + [0, 4] + [9] * 12),
    ("small_run_in_valley", 14250, [9] * 12 + [2, 9, 9, 1, 3] + [9] * 12),
    ("argmin_ties", 20250, [9] * 12 + [2, 1, 1] + [9] * 12 + [1, 5] + [9] * 12),
    ("trailing_bin", 12750, [7] * 12 + [1] + [7] * 12 + [0]),
    ("cutoff_equal", 10250, [10] * 10 + [2] + [10] * 10),
]


def detect_cases(ref):
    out = {}
    res = 500
    args = make_args(correct_resolution=res)
    assert all(length == (len(c) - 1) * res + 250 for _n, length, c in FUNCTION_CASES)
    cov_dict = {name: np.array(c, dtype=np.int32) for name, _l, c in FUNCTION_CASES}
    fa = {name: [None, length, 1] for name, length, _c in FUNCTION_CASES}
    got = ref.detect_break_points(cov_dict, fa, args)
    out["names"] = np.array([n for n, _l, _c in FUNCTION_CASES])
    out["lengths"] = np.array([l for _n, l, _c in FUNCTION_CASES], dtype=np.int64)
    out["cov_json"] = np.array(json.dumps([list(c) for _n, _l, c in FUNCTION_CASES]))
    out["breaks_json"] = np.array(json.dumps({k: [[int(p), int(c)] for p, c in v] for k, v in got.items()}))
    np.savez_compressed(os.path.join(HERE, "correct_detect.npz"), **out)
    print("correct_detect:", {k: v for k, v in got.items()})


def record_rounds(ref):
    """Wrap detect_break_points: every round's coverage dict (copied) and breakpoints."""
    rounds = []
    orig = ref.detect_break_points

    def wrapped(ctg_cov_dict, fa_dict, args):
        got = orig(ctg_cov_dict, fa_dict, args)
        rounds.append(({k: v.copy() for k, v in ctg_cov_dict.items()}, {k: list(v) for k, v in got.items()}))
        return got

    ref.detect_break_points = wrapped
    return rounds, lambda: setattr(ref, "detect_break_points", orig)


def pairs_case(ref, tag, nchr, n_contigs, mean_len, n_pairs, n_joins, span, seed, argkw):
    from haphic_b200 import synth
    group = 3 if "g3" in tag else 2
    gap = 0 if tag.endswith("nogap") else 1000
    asm, pairs, junctions = synth.chimera_case(nchr, n_contigs, mean_len, n_pairs, n_joins, span, seed, group=group, gap=gap)
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        cwd = os.getcwd()
        os.chdir(tmp)
        try:
            synth.write_fasta(asm, "asm.fa", seed=seed + 5)
            synth.write_pairs(asm, pairs, "aln.pairs")
            args = make_args(fasta="asm.fa", alignments="aln.pairs", aln_format="pairs", nchrs=nchr, **argkw)
            fa_dict = ref.parse_fasta("asm.fa", RE=args.RE)
            cov, links = ref.parse_pairs_for_correction(fa_dict, args)
            rounds, restore = record_rounds(ref)
            try:
                nbroken, final_pos, final_frag = ref.correct_assembly(cov, links, fa_dict, dict(), args)
            finally:
                restore()
            rj = []
            for cdict, brk in rounds:
                rj.append({"names": list(cdict.keys()), "cov": [v.tolist() for v in cdict.values()],
                           "breaks": [[k, [[int(p), int(c)] for p, c in v]] for k, v in brk.items()]})
            out["rounds_json"] = np.array(json.dumps(rj))
            out["fa_json"] = np.array(json.dumps([[k, int(v[1]), int(v[2])] for k, v in fa_dict.items()]))
            out["final_pos_json"] = np.array(json.dumps({k: [int(x) for x in v] for k, v in final_pos.items()}))
            out["final_frag_json"] = np.array(json.dumps(final_frag))
            out["nbroken"] = np.int64(nbroken)
            with open("corrected_ctgs.txt") as f:
                out["corrected_ctgs"] = np.array(f.read())
            import hashlib
            with open("corrected_asm.fa") as f:
                out["corrected_asm_sha1"] = np.array(hashlib.sha1(f.read().encode()).hexdigest())
            out["case_json"] = np.array(json.dumps([nchr, n_contigs, mean_len, n_pairs, n_joins, span, seed, group, gap]))
            out["argkw"] = np.array(json.dumps(argkw))
        finally:
            os.chdir(cwd)
    np.savez_compressed(os.path.join(HERE, "correct_{}.npz".format(tag)), **out)
    print("correct_{}: rounds={} breaks/round={} nbroken={} fa={}".format(
        tag, len(rounds), [len(b) for _c, b in rounds], nbroken, len(fa_dict)))


def run_case(ref, tag, nchr, n_contigs, mean_len, n_pairs, n_joins, span, seed, group, argkw):
    from haphic_b200 import synth
    import hashlib
    import pickle
    asm, pairs, junctions = synth.chimera_case(nchr, n_contigs, mean_len, n_pairs, n_joins, span, seed, group=group)
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        cwd = os.getcwd()
        os.chdir(tmp)
        try:
            synth.write_fasta(asm, "asm.fa", seed=seed + 5)
            synth.write_pairs(asm, pairs, "aln.pairs")
            args = make_args(fasta="asm.fa", alignments="aln.pairs", nchrs=nchr, **argkw)
            ref.INTEL_MKL = True
            ref.dot_product_mkl = lambda a, b: a @ b
            ref.run(args, log_file="HapHiC_cluster.log")
            files = {}
            for root, _dirs, fnames in os.walk("."):
                for fn in fnames:
                    p = os.path.join(root, fn)[2:]
                    if p.endswith(".txt") and (p.startswith("inflation_") or p == "corrected_ctgs.txt"):
                        with open(p) as f:
                            files[p] = f.read()
            with open("HapHiC_cluster.log") as f:
                log = f.read()
            out["recommend_lines"] = np.array([ln.split("] ", 1)[1] for ln in log.splitlines() if "[recommend_inflation]" in ln])
            out["mcl_lines"] = np.array([ln.split("] ", 1)[1] for ln in log.splitlines() if "[mcl]" in ln])
            with open("full_links.pkl", "rb") as f:
                full = pickle.load(f)
            with open("HT_links.pkl", "rb") as f:
                HT = pickle.load(f)
            # canonical JSON of the dicts in insertion order (full) / sorted (HT), kept as digests
            out["full_links_sha1"] = np.array(hashlib.sha1(json.dumps([[a, b, int(v)] for (a, b), v in full.items()]).encode()).hexdigest())
            out["HT_links_sha1"] = np.array(hashlib.sha1(json.dumps(sorted([[a, b, int(v)] for (a, b), v in HT.items()])).encode()).hexdigest())
            with open("paired_links.clm") as f:
                out["clm_sha1"] = np.array(hashlib.sha1(f.read().encode()).hexdigest())
            with open("alignments.bed") as f:
                out["bed_sha1"] = np.array(hashlib.sha1(f.read().encode()).hexdigest())
            out["asm_is_link"] = np.bool_(os.path.islink("corrected_asm.fa"))
            with open("corrected_asm.fa") as f:
                out["corrected_asm_sha1"] = np.array(hashlib.sha1(f.read().encode()).hexdigest())
            out["files_json"] = np.array(json.dumps(files, sort_keys=True))
            out["case_json"] = np.array(json.dumps([nchr, n_contigs, mean_len, n_pairs, n_joins, span, seed, group]))
            out["argkw"] = np.array(json.dumps(argkw, sort_keys=True))
        finally:
            os.chdir(cwd)
    np.savez_compressed(os.path.join(HERE, "correct_{}.npz".format(tag)), **out)
    print("correct_{}: {} files, recommend={}".format(tag, len(files), out["recommend_lines"].tolist()))


def main():
    sys.modules["portion"] = _portion
    ref = import_reference()
    only = set(sys.argv[1:])
    if not only or "detect" in only:
        detect_cases(ref)
    for case in PAIRS_CASES:
        if not only or case[0] in only:
            pairs_case(ref, *case)
    for case in RUN_CASES:
        if not only or case[0] in only:
            run_case(ref, *case)


if __name__ == "__main__":
    main()
