#!/usr/bin/env python3
"""Golden fixtures for `haphic cluster --gfa` (hifiasm read depths and phasing), made by the REFERENCE's own code:

    python tests/golden/make_gfa_golden.py

Imports scripts/HapHiC_cluster.py of the reference unmodified, the way make_golden.py does (same stubs, PYTHONHASHSEED=0),
writes one GFA file per haplotype with synth.write_gfa and runs the reference's run() on them.  Every run freezes its output
files, the log lines of the functions --gfa touches, the pickles (SHA-1 of the file and the items in insertion order with
their value types), and the inputs / outputs of filter_fragments and reduce_inter_hap_HiC_links, recorded by wrapping them
at run time.  Writes tests/golden/gfa_*.npz."""

import hashlib
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

import _portion                 # functional stand-in for `portion`, installed before the reference is imported
from make_golden import import_reference, make_args

SWEEP = dict(min_inflation=1.4, max_inflation=2.2, inflation_step=0.4)
# (tag, nchr, n_contigs, mean_len, n_pairs, seed, ploidy, n_gfa, chimeras, argkw); nchr counts haplotype chromosomes
RUN_CASES = [
    ("w1", 4, 160, 50000, 150000, 1201, 2, 2, 0, dict(Nx=100, bin_size=0, **SWEEP)),
    ("w05_norm", 4, 160, 50000, 150000, 1202, 2, 2, 0, dict(Nx=100, bin_size=0, phasing_weight=0.5, normalize_by_nlinks=True,
                                                         **SWEEP)),
    ("one_x", 4, 160, 50000, 150000, 1203, 2, 1, 0, dict(Nx=100, bin_size=0, **SWEEP)),
    ("one_frac", 4, 160, 50000, 150000, 1203, 2, 1, 0, dict(Nx=100, bin_size=0, read_depth_upper="0.9", **SWEEP)),
    ("bins", 4, 60, 300000, 150000, 1204, 2, 2, 0, dict(Nx=100, bin_size=120, flank=60, **SWEEP)),
    ("allelic", 4, 160, 50000, 150000, 1205, 2, 2, 0, dict(Nx=100, bin_size=0, remove_allelic_links=2, **SWEEP)),
    ("correct", 4, 160, 50000, 150000, 1206, 2, 2, 6, dict(Nx=100, bin_size=0, correct_nrounds=2, **SWEEP)),
    ("correct_qv", 4, 160, 50000, 150000, 1206, 2, 2, 6, dict(correct_nrounds=2, quick_view=True)),
]
LOGGED = ("parse_gfa", "filter_fragments", "reduce_inter_hap_HiC_links", "recommend_inflation", "mcl", "correct_assembly")


def sha(data):
    return hashlib.sha1(data if isinstance(data, bytes) else data.encode()).hexdigest()


def blob(obj, sort_keys=False):
    """JSON of ``obj`` as UTF-8 bytes (uint8 array): a numpy str array would store 4 bytes per character."""
    return np.frombuffer(json.dumps(obj, sort_keys=sort_keys).encode(), np.uint8)


def typed_items(d):
    """[[key..., repr(value)], ...] in insertion order: repr keeps int / float apart (2 vs 2.0)."""
    return [list(k) + [repr(v)] if isinstance(k, tuple) else [k, repr(v)] for k, v in d.items()]


def run_case(ref, tag, nchr, n_contigs, mean_len, n_pairs, seed, ploidy, n_gfa, chimeras, argkw):
    out = {}
    rec = {}
    orig_filter, orig_reduce = ref.filter_fragments, ref.reduce_inter_hap_HiC_links

    def filter_wrap(*a):
        got = orig_filter(*a)
        (nx, re_sites, cutoff, frag_links, d_lo, d_hi, top, rs_up, rs_hard, flank, depth, depth_up, wl) = a
        rec["filter_in"] = dict(Nx_frag_set=list(nx), RE_site_dict=re_sites, RE_site_cutoff=cutoff,
                                frag_link_dict=dict(frag_links), density_lower=d_lo, density_upper=d_hi, topN=top,
                                rank_sum_upper=rs_up, rank_sum_hard_cutoff=rs_hard, flank_link_dict=typed_items(flank),
                                read_depth_dict={k: list(v) for k, v in depth.items()}, read_depth_upper=depth_up)
        rec["filter_out"] = sorted(got)
        return got

    def reduce_wrap(link_dict, read_depth_dict, w, target="flank_link_dict"):
        before = typed_items(link_dict)
        orig_reduce(link_dict, read_depth_dict, w, target=target)
        rec["reduce_" + target] = dict(before=before, after=typed_items(link_dict), weight=w,
                                      hap={k: v[0] for k, v in read_depth_dict.items()})

    ref.filter_fragments, ref.reduce_inter_hap_HiC_links = filter_wrap, reduce_wrap
    with tempfile.TemporaryDirectory() as tmp:
        cwd = os.getcwd()
        os.chdir(tmp)
        try:
            from haphic_b200 import synth
            gfa = synth.gfa_case(nchr, n_contigs, mean_len, n_pairs, seed, ploidy, n_gfa, chimeras, tmp)
            args = make_args(fasta=os.path.join(tmp, "asm.fa"), alignments=os.path.join(tmp, "aln.pairs"), nchrs=nchr,
                             gfa=",".join(gfa), **argkw)
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
                    elif p.startswith("corrected_") and p.endswith(".gfa"):
                        files[p] = ("link:" + os.path.basename(os.readlink(p))) if os.path.islink(p) else open(p).read()
                    elif p.endswith((".pkl", ".clm", ".bed")) or p.startswith("corrected_"):
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
            if not argkw.get("quick_view"):
                with open("full_links.pkl", "rb") as f:
                    out["full_links_items"] = blob(typed_items(pickle.load(f)))
            out["files_json"] = blob(files, sort_keys=True)
            out["digests_json"] = blob(digests, sort_keys=True)
            out["record_json"] = blob(rec)
            out["argkw"] = blob(argkw, sort_keys=True)
            out["case"] = np.array([nchr, n_contigs, mean_len, n_pairs, seed, ploidy, n_gfa, chimeras], dtype=np.int64)
        finally:
            os.chdir(cwd)
            ref.filter_fragments, ref.reduce_inter_hap_HiC_links = orig_filter, orig_reduce
    np.savez_compressed(os.path.join(HERE, "gfa_{}.npz".format(tag)), **out)
    print("gfa_{}: {} files, {} log lines, recorded {}".format(tag, len(files), len(lines), sorted(rec)))


def parse_cases(ref):
    """parse_gfa on the error / warning inputs: (tag, message or None, warning lines)."""
    from haphic_b200 import synth
    asm = synth.make_assembly(2, 8, 20000, seed=1300)
    fa = {n: [None, int(ln), 1] for n, ln in zip(asm.names, asm.lengths.tolist())}
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        cases = {}
        gfa = [os.path.join(tmp, "ok{}.gfa".format(k)) for k in range(2)]
        synth.write_gfa(asm, gfa, seed=1301)
        cases["ok"] = gfa
        bad = os.path.join(tmp, "bad_len.gfa")
        with open(gfa[0]) as f, open(bad, "w") as g:
            g.write(f.read().replace("LN:i:", "LN:i:1", 1))
        cases["bad_len"] = [bad, gfa[1]]
        cases["missing"] = [gfa[0]]
        extra = [os.path.join(tmp, "ex{}.gfa".format(k)) for k in range(2)]
        synth.write_gfa(asm, extra, seed=1301, extra=("unplaced_1", "unplaced_2"))
        cases["extra"] = extra
        for tag, files in cases.items():
            logs = []
            handler = logging.Handler()
            handler.emit = lambda r: logs.append("{} {}".format(r.levelname, r.getMessage()))
            ref.logger.addHandler(handler)
            try:
                got = ref.parse_gfa(files, fa)
                res = dict(result={k: list(v) for k, v in got.items()}, order=list(got), error=None)
            except RuntimeError as e:
                res = dict(result=None, order=None, error=str(e))
            finally:
                ref.logger.removeHandler(handler)
            res["logs"] = logs
            res["files"] = {os.path.basename(p): open(p).read() for p in files}
            res["file_order"] = [os.path.basename(p) for p in files]
            out[tag] = res
    out["fa"] = {n: v[1] for n, v in fa.items()}
    np.savez_compressed(os.path.join(HERE, "gfa_parse.npz"), parse_json=blob(out))
    print("gfa_parse:", {k: (v["error"] is not None, len(v["logs"])) for k, v in out.items() if k != "fa"})


def main():
    sys.modules["portion"] = _portion
    ref = import_reference()
    only = set(sys.argv[1:])
    if not only or "parse" in only:
        parse_cases(ref)
    for case in RUN_CASES:
        if not only or case[0] in only:
            run_case(ref, *case)


if __name__ == "__main__":
    main()
