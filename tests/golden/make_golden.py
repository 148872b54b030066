#!/usr/bin/env python3
"""Generate the golden fixtures under tests/golden/ by running the REFERENCE's own code.

Run in the build container only (needs /root/reference, which does not exist
on the GPU box):

    python tests/golden/make_golden.py

What it does
------------
* installs import stubs for ``pysam`` and ``portion`` (neither is installed and
  neither is touched on the .pairs path; SURVEY.md section 8c), imports
  ``/root/reference/scripts/HapHiC_cluster.py`` UNMODIFIED,
* fabricates small inputs with ``haphic_b200.synth`` (seeded),
* calls the reference's functions on them and freezes inputs + outputs into
  ``tests/golden/*.npz`` (+ a JSON with the library versions used),
* for the sparse MCL path, ``dot_product_mkl`` (Intel MKL, not installed) is
  replaced by SciPy's ``a @ b`` -- stated in the fixture metadata.

The interpreter re-executes itself with PYTHONHASHSEED=0 because the reference
iterates sets of strings (HapHiC_cluster.py:357, 753).
"""

import json
import os
import sys
import tempfile
import types

if os.environ.get("PYTHONHASHSEED") != "0":
    os.environ["PYTHONHASHSEED"] = "0"
    os.execv(sys.executable, [sys.executable] + sys.argv)

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference/scripts"
sys.path.insert(0, REPO)

import numpy as np
import time
import scipy
import scipy.sparse as sp
import sklearn


def import_reference():
    pysam = types.ModuleType("pysam")
    pysam.set_verbosity = lambda *_a, **_k: 0
    pysam.AlignmentFile = None
    portion = types.ModuleType("portion")
    portion.closed = lambda *_a, **_k: None
    portion.empty = lambda *_a, **_k: None
    sys.modules.setdefault("pysam", pysam)
    sys.modules.setdefault("portion", portion)
    sys.path.insert(0, REF)
    import HapHiC_cluster as ref
    return ref


def make_args(**kw):
    """argparse.Namespace with the reference's defaults (HapHiC_cluster.py:2530-2735)."""
    import argparse
    d = dict(fasta=None, alignments=None, nchrs=4, aln_format="auto", RE="GATC", quick_view=False, gfa=None, ul=None,
             correct_nrounds=0, correct_resolution=500, median_cov_ratio=0.2, region_len_ratio=0.1,
             min_region_cutoff=5000, Nx=80, RE_site_cutoff=5, density_lower="0.2X", density_upper="1.9X",
             read_depth_upper="1.5X", topN=10, rank_sum_hard_cutoff=0, rank_sum_upper="1.5X",
             remove_allelic_links=0, concordance_ratio_cutoff=0.2, nwindows=50, remove_concentrated_links=False,
             max_read_pairs=200, min_read_pairs=20, phasing_weight=1.0, min_ul_mapq=30,
             min_ul_alignment_length=10000, max_distance_to_end=100, max_overlap_ratio=0.5, max_gap_len=10000,
             min_ul_support=2, bin_size=-1, flank=500, normalize_by_nlinks=False, expansion=2, min_inflation=1.1,
             max_inflation=3.0, inflation_step=0.1, max_iter=200, pruning=0.0001, skip_clustering=False,
             threads=8, dense_matrix=False, verbose=False)
    d.update(kw)
    return argparse.Namespace(**d)


def dict_pairs_to_arrays(d, name_to_id, value_dtype):
    keys = np.array([(name_to_id[a], name_to_id[b]) for (a, b) in d.keys()], dtype=np.int32).reshape(-1, 2)
    vals = np.array(list(d.values()), dtype=value_dtype)
    return keys, vals


def csc_arrays(m, prefix):
    m = sp.csc_matrix(m)
    m.sort_indices()
    return {prefix + "_indptr": m.indptr.astype(np.int64), prefix + "_indices": m.indices.astype(np.int32),
            prefix + "_data": m.data.astype(np.float32)}


def link_case(ref, tag, nchr, n_contigs, mean_len, n_pairs, flank, Nx, seed, normalize=False):
    """Golden for link counting (a3), normalisation (a6), filter (a7/a8), dict_to_matrix (a10)."""
    from haphic_b200 import synth
    asm = synth.make_assembly(nchr, n_contigs, mean_len, seed=seed)
    pairs = synth.make_pairs(asm, n_pairs, seed=seed + 1).numpy()
    # sprinkle records naming a contig that is absent from the FASTA (skipped at 1625)
    rng = np.random.default_rng(seed + 2)
    ghost_rows = rng.choice(n_pairs, size=max(1, n_pairs // 200), replace=False)
    ghost_side = rng.integers(0, 2, size=len(ghost_rows))
    names_ext = asm.names + ["ghost_ctg"]
    ghost_id = asm.n
    pairs_ext = pairs.copy()
    for r, s in zip(ghost_rows.tolist(), ghost_side.tolist()):
        pairs_ext[r, 2 * s] = ghost_id
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        cwd = os.getcwd()
        os.chdir(tmp)
        try:
            fasta = os.path.join(tmp, "asm.fa")
            pfile = os.path.join(tmp, "aln.pairs")
            synth.write_fasta(asm, fasta, seed=seed + 3)
            ext = synth.Assembly(names_ext, None, None, None, None, asm.chrom_len, asm.nchr)
            synth.write_pairs(ext, pairs_ext, pfile)
            args = make_args(fasta=fasta, alignments=pfile, nchrs=nchr, flank=flank, Nx=Nx, bin_size=0,
                             normalize_by_nlinks=normalize, aln_format="pairs")
            fa_dict = ref.parse_fasta(fasta, RE=args.RE)
            pos_t, dist_t = ref.determine_int_type(fa_dict)
            _, bin_set, bin_size, frag_len_dict, Nx_frag_set, RE_site_dict, split_ctg_set = ref.stat_fragments(
                fa_dict, args.RE, dict(), set(), nchrs=nchr, flank=flank, Nx=Nx, bin_size=0)
            assert not split_ctg_set
            alignments = ref.pairs_generator_inter_ctgs(pfile, "pairs")
            full, flank_d, HT, clm, ctg_links, _coord = ref.parse_alignments_for_ctgs(
                alignments, fa_dict, args, frag_len_dict, Nx_frag_set, pos_t, dist_t)
            name_to_id = {n: i for i, n in enumerate(asm.names)}
            out["names"] = np.array(asm.names)
            out["lengths"] = asm.lengths
            out["RE_sites"] = np.array([fa_dict[n][2] for n in asm.names], dtype=np.int64)
            out["RE_site_dict"] = np.array([RE_site_dict[n] for n in asm.names], dtype=np.int64)
            out["pairs"] = pairs_ext.astype(np.int32)
            out["ghost_id"] = np.int32(ghost_id)
            out["flank_kb"] = np.int64(flank)
            out["Nx"] = np.int64(Nx)
            out["in_nx"] = np.array([n in Nx_frag_set for n in asm.names], dtype=np.uint8)
            out["full_keys"], out["full_vals"] = dict_pairs_to_arrays(full, name_to_id, np.int64)
            out["flank_keys"], out["flank_vals"] = dict_pairs_to_arrays(flank_d, name_to_id, np.int64)
            # HT dict: keys are names with _H/_T suffix; encode as (id_i, t_i, id_j, t_j)
            hk = []
            for (a, b) in HT.keys():
                hk.append((name_to_id[a[:-2]], int(a.endswith("_T")), name_to_id[b[:-2]], int(b.endswith("_T"))))
            out["HT_keys"] = np.array(hk, dtype=np.int32).reshape(-1, 4)
            out["HT_vals"] = np.array(list(HT.values()), dtype=np.int64)
            out["ctg_link_ids"] = np.array([name_to_id[k] for k in ctg_links.keys()], dtype=np.int32)
            out["ctg_link_vals"] = np.array(list(ctg_links.values()), dtype=np.int64)
            ck, co, cv = [], [0], []
            for (a, b), arr in clm.items():
                ck.append((name_to_id[a], name_to_id[b]))
                cv.extend(arr.tolist())
                co.append(len(cv))
            out["clm_keys"] = np.array(ck, dtype=np.int32).reshape(-1, 2)
            out["clm_offsets"] = np.array(co, dtype=np.int64)
            out["clm_vals"] = np.array(cv, dtype=np.int64)
            ref.output_clm(clm)
            with open("paired_links.clm") as f:
                out["clm_text"] = np.array(f.read())
            if normalize:
                ref.normalize_by_nlinks(flank_d, ctg_links)
                out["flank_norm_vals"] = np.array(list(flank_d.values()), dtype=np.float64)
            filtered = ref.filter_fragments(
                Nx_frag_set, RE_site_dict, args.RE_site_cutoff, ctg_links, args.density_lower, args.density_upper,
                args.topN, args.rank_sum_upper, args.rank_sum_hard_cutoff, flank_d, dict(), args.read_depth_upper,
                set())
            out["filtered"] = np.array([n in filtered for n in asm.names], dtype=np.uint8)
            matrix, frag_index = ref.dict_to_matrix(flank_d, filtered, dense_matrix=False, add_self_loops=True)
            out["matrix_index"] = np.array([frag_index.get(n, -1) for n in asm.names], dtype=np.int32)
            out.update(csc_arrays(matrix, "link"))
        finally:
            os.chdir(cwd)
    np.savez_compressed(os.path.join(HERE, "links_{}.npz".format(tag)), **out)
    print("links_{}: n={} P={} nnz_full={} nnz_flank={} kept={}".format(
        tag, asm.n, n_pairs, len(out["full_vals"]), len(out["flank_vals"]), int(out["filtered"].sum())))
    return matrix


def link_case_bins(ref, tag, nchr, n_contigs, mean_len, n_pairs, flank, Nx, bin_kb, seed):
    """Golden for parse_alignments (a4): contigs longer than bin_size are split into bins."""
    from haphic_b200 import synth
    asm = synth.make_assembly(nchr, n_contigs, mean_len, seed=seed)
    pairs = synth.make_pairs(asm, n_pairs, seed=seed + 1).numpy()
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        cwd = os.getcwd()
        os.chdir(tmp)
        try:
            fasta = os.path.join(tmp, "asm.fa")
            pfile = os.path.join(tmp, "aln.pairs")
            synth.write_fasta(asm, fasta, seed=seed + 3)
            synth.write_pairs(asm, pairs, pfile)
            args = make_args(fasta=fasta, alignments=pfile, nchrs=nchr, flank=flank, Nx=Nx, bin_size=bin_kb, aln_format="pairs")
            fa_dict = ref.parse_fasta(fasta, RE=args.RE)
            pos_t, dist_t = ref.determine_int_type(fa_dict)
            _, bin_set, bin_size, frag_len_dict, Nx_frag_set, RE_site_dict, split_ctg_set = ref.stat_fragments(
                fa_dict, args.RE, dict(), set(), nchrs=nchr, flank=flank, Nx=Nx, bin_size=bin_kb)
            assert split_ctg_set
            alignments = ref.pairs_generator(pfile, "pairs")
            full, flank_d, HT, clm, frag_links, _coord, _c2f = ref.parse_alignments(
                alignments, fa_dict, args, bin_size, frag_len_dict, Nx_frag_set, split_ctg_set, pos_t, dist_t)
            # fragment ids: FASTA order, bins of a split contig in bin order
            frag_names = []
            frag_base = [0]
            import math
            for ctg, info in fa_dict.items():
                if ctg in split_ctg_set:
                    frag_names += ["{}_bin{}".format(ctg, k + 1) for k in range(math.ceil(info[1] / bin_size))]
                else:
                    frag_names.append(ctg)
                frag_base.append(len(frag_names))
            fid = {n: i for i, n in enumerate(frag_names)}
            cid = {n: i for i, n in enumerate(asm.names)}
            out["names"] = np.array(asm.names)
            out["lengths"] = asm.lengths
            out["pairs"] = pairs.astype(np.int32)
            out["flank_kb"] = np.int64(flank)
            out["Nx"] = np.int64(Nx)
            out["bin_kb"] = np.int64(bin_kb)
            out["bin_size"] = np.int64(bin_size)
            out["frag_names"] = np.array(frag_names)
            out["frag_base"] = np.array(frag_base, dtype=np.int32)
            out["frag_len"] = np.array([frag_len_dict[f] for f in frag_names], dtype=np.int64)
            out["frag_in_nx"] = np.array([f in Nx_frag_set for f in frag_names], dtype=np.uint8)
            out["frag_RE"] = np.array([RE_site_dict[f] for f in frag_names], dtype=np.int64)
            out["full_keys"], out["full_vals"] = dict_pairs_to_arrays(full, cid, np.int64)
            out["flank_keys"], out["flank_vals"] = dict_pairs_to_arrays(flank_d, fid, np.int64)
            hk = [(cid[a[:-2]], int(a.endswith("_T")), cid[b[:-2]], int(b.endswith("_T"))) for (a, b) in HT.keys()]
            out["HT_keys"] = np.array(hk, dtype=np.int32).reshape(-1, 4)
            out["HT_vals"] = np.array(list(HT.values()), dtype=np.int64)
            out["frag_link_ids"] = np.array([fid[k] for k in frag_links.keys()], dtype=np.int32)
            out["frag_link_vals"] = np.array(list(frag_links.values()), dtype=np.int64)
            ref.output_clm(clm)
            with open("paired_links.clm") as f:
                out["clm_text"] = np.array(f.read())
        finally:
            os.chdir(cwd)
    np.savez_compressed(os.path.join(HERE, "links_{}.npz".format(tag)), **out)
    print("links_{}: n_ctg={} n_frag={} P={} nnz_full={} nnz_flank={}".format(
        tag, asm.n, len(frag_names), n_pairs, len(out["full_vals"]), len(out["flank_vals"])))


def link_case_bins_edges(ref, tag, n_rec, flanks_kb, Nx, seed):
    """Golden for parse_alignments at the edges of binning (tests/frag_edges.py): one stream counted with each flank
    size, and the single records of frag_edges.SINGLE each parsed on its own with the outcome the reference gives it
    (skipped, counted or a KeyError, which ends the reference's run)."""
    import math
    from tests import frag_edges as E
    names = E.names()
    rng = np.random.default_rng(seed)
    pairs = E.stream(n_rec, seed + 1)
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        cwd = os.getcwd()
        os.chdir(tmp)
        try:
            fasta = os.path.join(tmp, "asm.fa")
            pfile = os.path.join(tmp, "aln.pairs")
            with open(fasta, "w") as f:
                for nm, ln in E.LAYOUT:
                    f.write(">{}\n{}\n".format(nm, "".join(np.array(list("ACGT"))[rng.integers(0, 4, ln)])))
            ext = names + [E.GHOST]

            def write_pairs(path, rec):
                with open(path, "w") as f:
                    f.write("## pairs format v1.0\n")
                    for r, (a, pa, b, pb) in enumerate(np.asarray(rec).tolist()):
                        f.write("r{}\t{}\t{}\t{}\t{}\t+\t-\n".format(r, ext[a], pa + 1, ext[b], pb + 1))

            write_pairs(pfile, pairs)
            fa_dict = ref.parse_fasta(fasta, RE="GATC")
            pos_t, dist_t = ref.determine_int_type(fa_dict)
            _, bin_set, bin_size, frag_len_dict, Nx_frag_set, RE_site_dict, split_ctg_set = ref.stat_fragments(
                fa_dict, "GATC", dict(), set(), nchrs=2, flank=flanks_kb[0], Nx=Nx, bin_size=E.BIN_KB)
            frag_names, frag_base = [], [0]
            for ctg, info in fa_dict.items():
                if ctg in split_ctg_set:
                    frag_names += ["{}_bin{}".format(ctg, k + 1) for k in range(math.ceil(info[1] / bin_size))]
                else:
                    frag_names.append(ctg)
                frag_base.append(len(frag_names))
            fid = {n: i for i, n in enumerate(frag_names)}
            cid = {n: i for i, n in enumerate(names)}
            out["names"] = np.array(names)
            out["lengths"] = E.lengths()
            out["pairs"] = pairs
            out["ghost_id"] = np.int32(len(names))
            out["Nx"] = np.int64(Nx)
            out["bin_size"] = np.int64(bin_size)
            out["flanks_kb"] = np.array(flanks_kb, np.int64)
            out["frag_names"] = np.array(frag_names)
            out["frag_base"] = np.array(frag_base, dtype=np.int32)
            out["frag_len"] = np.array([frag_len_dict[f] for f in frag_names], dtype=np.int64)
            out["frag_in_nx"] = np.array([f in Nx_frag_set for f in frag_names], dtype=np.uint8)
            for fk in flanks_kb:
                args = make_args(fasta=fasta, alignments=pfile, nchrs=2, flank=fk, Nx=Nx, bin_size=E.BIN_KB,
                                 aln_format="pairs", remove_allelic_links=2)
                full, flank_d, HT, _clm, frag_links, _coord, c2f = ref.parse_alignments(
                    ref.pairs_generator(pfile, "pairs"), fa_dict, args, bin_size, frag_len_dict, Nx_frag_set, split_ctg_set,
                    pos_t, dist_t)
                p = "flank{}_".format(fk)
                out[p + "keys"], out[p + "vals"] = dict_pairs_to_arrays(flank_d, fid, np.int64)
                out[p + "frag_link_ids"] = np.array([fid[k] for k in frag_links.keys()], dtype=np.int32)
                out[p + "frag_link_vals"] = np.array(list(frag_links.values()), dtype=np.int64)
            # full / HT / ctg_pair_to_frag do not depend on the flank size
            out["full_keys"], out["full_vals"] = dict_pairs_to_arrays(full, cid, np.int64)
            hk = [(cid[a[:-2]], int(a.endswith("_T")), cid[b[:-2]], int(b.endswith("_T"))) for (a, b) in HT.keys()]
            out["HT_keys"] = np.array(hk, dtype=np.int32).reshape(-1, 4)
            out["HT_vals"] = np.array(list(HT.values()), dtype=np.int64)
            out["c2f_json"] = np.array(json.dumps(sorted([[a, b, sorted(map(list, v))] for (a, b), v in c2f.items()])))
            single, outcome = E.single_records(), []
            for k in range(len(single)):
                rec = single[k:k + 1]
                sfile = os.path.join(tmp, "single{}.pairs".format(k))
                write_pairs(sfile, rec)
                try:
                    _f, _fl, _h, _c, _t, _co, c2f1 = ref.parse_alignments(
                        ref.pairs_generator(sfile, "pairs"), fa_dict, args, bin_size, frag_len_dict, Nx_frag_set,
                        split_ctg_set, pos_t, dist_t)
                    outcome.append(E.COUNTED if c2f1 else E.SKIPPED)
                except KeyError:
                    outcome.append(E.RAISES)
            out["single_recs"] = single
            out["single_outcome"] = np.array(outcome, np.int8)
        finally:
            os.chdir(cwd)
    np.savez_compressed(os.path.join(HERE, "links_{}.npz".format(tag)), **out)
    print("links_{}: n_ctg={} n_frag={} P={} nnz_full={} nnz_flank={} single outcomes={}".format(
        tag, len(names), len(frag_names), n_rec, len(out["full_vals"]),
        [len(out["flank{}_vals".format(fk)]) for fk in flanks_kb], out["single_outcome"].tolist()))


def mcl_case(ref, tag, link_matrix, inflations, pruning=1e-4, expansion=2, max_iter=200, keep_iters=4):
    """Golden for MCL (a11-a15): first normalisation, pre-expansion, per-iteration matrices, clusters."""
    from sklearn.preprocessing import normalize
    ref.INTEL_MKL = True
    ref.dot_product_mkl = lambda a, b: a @ b           # SciPy SpGEMM stands in for MKL
    out = {}
    link = sp.csc_matrix(link_matrix, dtype=np.float32)
    out.update(csc_arrays(link, "link"))
    m0 = normalize(link, norm="l1", axis=0)
    out.update(csc_arrays(m0, "m0"))
    m1 = ref.mkl_matrix_power(m0, expansion)
    out["m1_dense"] = np.asarray(m1.todense(), dtype=np.float32)
    out["inflations"] = np.array(inflations, dtype=np.float64)
    out["pruning"] = np.float64(pruning)
    out["expansion"] = np.int64(expansion)
    import logging
    import io
    for r in inflations:
        # iteration count = what the reference logs
        stream = io.StringIO()
        h = logging.StreamHandler(stream)
        ref.logger.addHandler(h)
        final = ref.mcl(m1, expansion, float(r), max_iter, pruning, False)
        ref.logger.removeHandler(h)
        msg = stream.getvalue()
        n_iter = int(msg.split("after ")[1].split(" rounds")[0])
        converged = "has converged" in msg
        key = "r{}".format(str(r).replace(".", "p"))
        out[key + "_niter"] = np.int64(n_iter)
        out[key + "_converged"] = np.bool_(converged)
        out.update(csc_arrays(final, key + "_final"))
        for k in range(1, keep_iters + 1):
            mk = ref.mcl(m1, expansion, float(r), k, pruning, False)
            out.update(csc_arrays(mk, key + "_iter{}".format(k)))
        clusters = ref.interpret_result(final, False)
        if clusters is None:
            out[key + "_clusters_valid"] = np.bool_(False)
        else:
            out[key + "_clusters_valid"] = np.bool_(True)
            lab = np.full(link.shape[0], -1, dtype=np.int32)
            for c in clusters:
                lab[list(c)] = min(c)
            out[key + "_labels"] = lab
        # dense path of the reference on the same input (iteration count must agree)
        stream = io.StringIO()
        h = logging.StreamHandler(stream)
        ref.logger.addHandler(h)
        m1d = np.asarray(m1.todense(), dtype=np.float32)
        ref.mcl(m1d, expansion, float(r), max_iter, pruning, True)
        ref.logger.removeHandler(h)
        out[key + "_niter_dense"] = np.int64(int(stream.getvalue().split("after ")[1].split(" rounds")[0]))
    np.savez_compressed(os.path.join(HERE, "mcl_{}.npz".format(tag)), **out)
    print("mcl_{}: n={} nnz={} iters={}".format(
        tag, link.shape[0], link.nnz, {str(r): int(out["r{}_niter".format(str(r).replace('.', 'p'))]) for r in inflations}))


def block_matrix(n_blocks, block, seed, noise=0.02):
    """Synthetic symmetric count matrix with ``n_blocks`` planted clusters (+ self loops = 1)."""
    rng = np.random.default_rng(seed)
    n = n_blocks * block
    a = np.zeros((n, n), dtype=np.float32)
    lab = np.repeat(np.arange(n_blocks), block)
    same = lab[:, None] == lab[None, :]
    dist = np.abs(np.arange(n)[:, None] - np.arange(n)[None, :])
    lam = np.where(same, 40.0 / (1.0 + dist), 0.0)
    counts = rng.poisson(lam).astype(np.float32)
    counts += (rng.random((n, n)) < noise) * rng.integers(1, 3, size=(n, n))
    counts = np.triu(counts, 1)
    a = counts + counts.T
    perm = rng.permutation(n)
    a = a[perm][:, perm]
    np.fill_diagonal(a, 1.0)
    return sp.csc_matrix(a, dtype=np.float32)


def allelic_case(ref, tag, nchr, ploidy, n_contigs, mean_len, n_pairs, frac, seed, concentrated=False, bin_kb=0, **argkw):
    """Golden for record_coord_pairs / the two ratios / remove_allelic_HiC_links (a9): nchr chromosomes x ploidy
    haplotypes, a fraction of the cis pairs re-mapped to the same locus of another haplotype."""
    from haphic_b200 import synth
    asm = synth.make_assembly(nchr * ploidy, n_contigs, mean_len, seed=seed)
    pairs = synth.make_pairs(asm, n_pairs, seed=seed + 1, homolog=(ploidy, frac)).numpy()
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        cwd = os.getcwd()
        os.chdir(tmp)
        try:
            fasta = os.path.join(tmp, "asm.fa")
            pfile = os.path.join(tmp, "aln.pairs")
            synth.write_fasta(asm, fasta, seed=seed + 3)
            synth.write_pairs(asm, pairs, pfile)
            args = make_args(fasta=fasta, alignments=pfile, nchrs=nchr * ploidy, bin_size=bin_kb, aln_format="pairs",
                             remove_allelic_links=ploidy, remove_concentrated_links=concentrated, **argkw)
            fa_dict = ref.parse_fasta(fasta, RE=args.RE)
            pos_t, dist_t = ref.determine_int_type(fa_dict)
            _, bin_set, bin_size, frag_len_dict, Nx_frag_set, RE_site_dict, split_ctg_set = ref.stat_fragments(
                fa_dict, args.RE, dict(), set(), nchrs=args.nchrs, flank=args.flank, Nx=args.Nx, bin_size=bin_kb)
            c2f = None
            if split_ctg_set:
                alignments = ref.pairs_generator(pfile, "pairs")
                full, flank_d, HT, clm, frag_links, coord, c2f = ref.parse_alignments(
                    alignments, fa_dict, args, bin_size, frag_len_dict, Nx_frag_set, split_ctg_set, pos_t, dist_t)
            else:
                alignments = ref.pairs_generator_inter_ctgs(pfile, "pairs")
                full, flank_d, HT, clm, frag_links, coord = ref.parse_alignments_for_ctgs(
                    alignments, fa_dict, args, frag_len_dict, Nx_frag_set, pos_t, dist_t)
            coord_json = [[a, b, (list(v) if isinstance(v, list) else None), (None if isinstance(v, list) else v.tolist())]
                          for (a, b), v in coord.items()]
            out["coord_json"] = np.array(json.dumps(coord_json))
            if c2f is not None:
                out["c2f_json"] = np.array(json.dumps(sorted([[a, b, sorted(map(list, v))] for (a, b), v in c2f.items() if a != b])))
            if concentrated:
                for pair, data in coord.items():
                    if isinstance(data, list):
                        full[pair] *= data[1]
            filtered = ref.filter_fragments(
                Nx_frag_set, RE_site_dict, args.RE_site_cutoff, frag_links, args.density_lower, args.density_upper,
                args.topN, args.rank_sum_upper, args.rank_sum_hard_cutoff, flank_d, dict(), args.read_depth_upper, set())
            out["full_before_json"] = np.array(json.dumps([[a, b, v] for (a, b), v in full.items()]))
            out["flank_before_json"] = np.array(json.dumps([[a, b, v] for (a, b), v in flank_d.items()]))
            out["filtered_json"] = np.array(json.dumps(sorted(filtered)))
            remaining = ref.remove_allelic_HiC_links(fa_dict, coord, full, args, flank_d, filtered, c2f if split_ctg_set else None)
            out["full_after_json"] = np.array(json.dumps([[a, b, v] for (a, b), v in full.items()]))
            out["flank_after_json"] = np.array(json.dumps([[a, b, v] for (a, b), v in flank_d.items()]))
            out["remaining_json"] = np.array(json.dumps(sorted(remaining)))
            out["names"] = np.array(asm.names)
            out["lengths"] = asm.lengths
            out["pairs"] = pairs.astype(np.int32)
            out["ploidy"] = np.int64(ploidy)
            out["bin_size"] = np.int64(bin_size if split_ctg_set else 0)
            out["argkw"] = np.array(json.dumps(dict(argkw, bin_size=bin_kb, remove_allelic_links=ploidy,
                                                    remove_concentrated_links=concentrated, nchrs=nchr * ploidy)))
            n_before, n_after = len(json.loads(str(out["full_before_json"]))), len(full)
        finally:
            os.chdir(cwd)
    np.savez_compressed(os.path.join(HERE, "allelic_{}.npz".format(tag)), **out)
    print("allelic_{}: contig pairs {} -> {} after removal, fragments {} -> {}, pairs with >= max_read_pairs: {}".format(
        tag, n_before, n_after, len(filtered), len(remaining), sum(1 for c in coord_json if c[2] is not None)))


def run_case(ref, tag, nchr, n_contigs, mean_len, n_pairs, seed, homolog=None, **argkw):
    """Golden for the whole `haphic cluster` run (boundary b): output files as text."""
    from haphic_b200 import synth
    asm = synth.make_assembly(nchr, n_contigs, mean_len, seed=seed)
    pairs = synth.make_pairs(asm, n_pairs, seed=seed + 1, homolog=homolog).numpy()
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        cwd = os.getcwd()
        os.chdir(tmp)
        try:
            fasta = os.path.join(tmp, "asm.fa")
            pfile = os.path.join(tmp, "aln.pairs")
            synth.write_fasta(asm, fasta, seed=seed + 3)
            synth.write_pairs(asm, pairs, pfile)
            args = make_args(fasta=fasta, alignments=pfile, nchrs=nchr, **argkw)
            ref.INTEL_MKL = True
            ref.dot_product_mkl = lambda a, b: a @ b
            ref.run(args, log_file="HapHiC_cluster.log")
            files = {}
            for root, _dirs, fnames in os.walk("."):
                for fn in fnames:
                    p = os.path.join(root, fn)[2:]
                    if p.endswith(".txt") and p.startswith("inflation_"):
                        with open(p) as f:
                            files[p] = f.read()
            with open("HapHiC_cluster.log") as f:
                log = f.read()
            rec = [ln.split("] ", 1)[1] for ln in log.splitlines() if "[recommend_inflation]" in ln]
            conv = [ln.split("] ", 1)[1] for ln in log.splitlines() if "[mcl]" in ln]
            import pickle
            with open("full_links.pkl", "rb") as f:
                full = pickle.load(f)
            with open("HT_links.pkl", "rb") as f:
                HT = pickle.load(f)
            with open("paired_links.clm") as f:
                out["clm_text"] = np.array(f.read())
            with open("alignments.bed") as f:
                bed = f.read()
            import hashlib
            out["bed_sha1"] = np.array(hashlib.sha1(bed.encode()).hexdigest())
            out["bed_head"] = np.array(bed[:2000])
            out["files_json"] = np.array(json.dumps(files, sort_keys=True))
            out["recommend_lines"] = np.array(rec)
            out["mcl_lines"] = np.array(conv)
            out["full_links_sorted"] = np.array(json.dumps(sorted([[a, b, int(v)] for (a, b), v in full.items()])))
            out["HT_links_sorted"] = np.array(json.dumps(sorted([[a, b, int(v)] for (a, b), v in HT.items()])))
            out["argkw"] = np.array(json.dumps(argkw, sort_keys=True))
            out["seed"] = np.int64(seed)
            out["shape"] = np.array([nchr, n_contigs, mean_len, n_pairs], dtype=np.int64)
            out["homolog"] = np.array(json.dumps(list(homolog) if homolog else None))
        finally:
            os.chdir(cwd)
    np.savez_compressed(os.path.join(HERE, "run_{}.npz".format(tag)), **out)
    print("run_{}: {} files, recommend={}".format(tag, len(files), rec))


def run_digest_case(ref, tag, nchr, n_contigs, mean_len, n_pairs, seed, homolog=None, **argkw):
    """Golden for a whole `haphic cluster` run at a size whose output files are too large to commit: SHA-1 digests of every
    output file / dict (canonical JSON of the sorted items), the machine-read log lines and the iteration counts."""
    import hashlib
    import pickle
    import re
    from haphic_b200 import synth
    asm = synth.make_assembly(nchr, n_contigs, mean_len, seed=seed)
    pairs = synth.make_pairs(asm, n_pairs, seed=seed + 1, homolog=homolog).numpy()
    out = {}

    def sha(text):
        return hashlib.sha1(text.encode()).hexdigest()

    with tempfile.TemporaryDirectory() as tmp:
        cwd = os.getcwd()
        os.chdir(tmp)
        try:
            synth.write_fasta(asm, "asm.fa", seed=seed + 3)
            synth.write_pairs(asm, pairs, "aln.pairs")
            args = make_args(fasta=os.path.join(tmp, "asm.fa"), alignments=os.path.join(tmp, "aln.pairs"), nchrs=nchr, **argkw)
            ref.INTEL_MKL = True
            ref.dot_product_mkl = lambda a, b: a @ b
            t0 = time.time()
            ref.run(args, log_file="HapHiC_cluster.log")
            out["reference_seconds"] = np.float64(time.time() - t0)
            files = {}
            for root, _dirs, fnames in os.walk("."):
                for fn in fnames:
                    p = os.path.join(root, fn)[2:]
                    if p.endswith(".txt") and p.startswith("inflation_"):
                        with open(p) as f:
                            files[p] = sha(f.read())
            with open("HapHiC_cluster.log") as f:
                log = f.read()
            out["recommend_lines"] = np.array([ln.split("] ", 1)[1] for ln in log.splitlines() if "[recommend_inflation]" in ln])
            out["mcl_lines"] = np.array([ln.split("] ", 1)[1] for ln in log.splitlines() if "[mcl]" in ln])
            with open("full_links.pkl", "rb") as f:
                full = pickle.load(f)
            with open("HT_links.pkl", "rb") as f:
                HT = pickle.load(f)
            out["n_full"] = np.int64(len(full))
            out["n_HT"] = np.int64(len(HT))
            out["full_links_sha1"] = np.array(sha(json.dumps(sorted([[a, b, int(v)] for (a, b), v in full.items()]))))
            out["full_links_order_sha1"] = np.array(sha(json.dumps([[a, b] for (a, b) in full.keys()])))
            out["HT_links_sha1"] = np.array(sha(json.dumps(sorted([[a, b, int(v)] for (a, b), v in HT.items()]))))
            with open("paired_links.clm") as f:
                out["clm_sha1"] = np.array(sha(f.read()))
            with open("alignments.bed") as f:
                out["bed_sha1"] = np.array(sha(f.read()))
            out["files_json"] = np.array(json.dumps(files, sort_keys=True))
            out["argkw"] = np.array(json.dumps(argkw, sort_keys=True))
            out["seed"] = np.int64(seed)
            out["shape"] = np.array([nchr, n_contigs, mean_len, n_pairs], dtype=np.int64)
            out["homolog"] = np.array(json.dumps(list(homolog) if homolog else None))
        finally:
            os.chdir(cwd)
    np.savez_compressed(os.path.join(HERE, "rundigest_{}.npz".format(tag)), **out)
    print("rundigest_{}: {} files, {:.0f} s, recommend={}".format(tag, len(files), float(out["reference_seconds"]),
                                                                 out["recommend_lines"].tolist()))


def main():
    """`make_golden.py` regenerates everything; `make_golden.py allelic run_allelic4` only the named groups."""
    ref = import_reference()
    only = set(sys.argv[1:])

    def want(group):
        return not only or group in only

    if want("links") or want("mcl"):
        m_a = link_case(ref, "a", nchr=3, n_contigs=60, mean_len=40000, n_pairs=30000, flank=500, Nx=100, seed=101)
        link_case(ref, "b", nchr=4, n_contigs=120, mean_len=60000, n_pairs=60000, flank=10, Nx=80, seed=202,
                  normalize=True)
    if want("mcl"):
        mcl_case(ref, "links_a", m_a, inflations=[1.2, 2.0, 3.0])
        mcl_case(ref, "block200", block_matrix(4, 50, seed=7), inflations=[1.1, 1.5, 2.0, 2.7])
        mcl_case(ref, "block600", block_matrix(6, 100, seed=9, noise=0.05), inflations=[1.4, 2.0], keep_iters=3)
    if want("run"):
        run_case(ref, "c1", nchr=4, n_contigs=200, mean_len=40000, n_pairs=150000, seed=303, Nx=100, bin_size=0)
        run_case(ref, "c1_nx80", nchr=4, n_contigs=200, mean_len=40000, n_pairs=150000, seed=303, Nx=80, bin_size=0,
                 min_inflation=1.2, max_inflation=2.0, inflation_step=0.2)
    if want("bins"):
        link_case_bins(ref, "bins", nchr=3, n_contigs=45, mean_len=300000, n_pairs=60000, flank=40, Nx=90, bin_kb=100, seed=404)
        run_case(ref, "bins", nchr=3, n_contigs=60, mean_len=350000, n_pairs=120000, seed=505, Nx=100, bin_size=120, flank=60,
                 min_inflation=1.4, max_inflation=2.2, inflation_step=0.4)
    if want("bins_edges"):
        link_case_bins_edges(ref, "bins_edges", n_rec=6000, flanks_kb=(1, 5), Nx=70, seed=1212)
    if want("allelic"):
        allelic_case(ref, "p2", nchr=3, ploidy=2, n_contigs=120, mean_len=60000, n_pairs=120000, frac=0.2, seed=606, Nx=100)
        allelic_case(ref, "p4", nchr=2, ploidy=4, n_contigs=160, mean_len=50000, n_pairs=200000, frac=0.3, seed=707, Nx=100,
                     concentrated=True, max_read_pairs=60)
        allelic_case(ref, "p4bins", nchr=2, ploidy=4, n_contigs=64, mean_len=300000, n_pairs=150000, frac=0.3, seed=808,
                     Nx=100, bin_kb=100, flank=40)
    if want("run_allelic4"):
        run_case(ref, "allelic4", nchr=8, n_contigs=160, mean_len=50000, n_pairs=200000, seed=909, homolog=(4, 0.3), Nx=100,
                 bin_size=0, remove_allelic_links=4, min_inflation=1.4, max_inflation=2.2, inflation_step=0.4)
    if "run_c4" in only:          # minutes of CPU: only on request
        run_digest_case(ref, "c4_10k", nchr=24, n_contigs=10000, mean_len=20000, n_pairs=5000000, seed=1111, homolog=(4, 0.3),
                        Nx=100, bin_size=0, remove_allelic_links=4, min_inflation=1.4, max_inflation=2.2, inflation_step=0.4)
        return
    meta = {"numpy": np.__version__, "scipy": scipy.__version__, "sklearn": sklearn.__version__,
            "python": sys.version.split()[0], "PYTHONHASHSEED": os.environ.get("PYTHONHASHSEED"),
            "reference": "zengxiaofei/HapHiC scripts/HapHiC_cluster.py (v1.0.7, commit 1f29080), imported unmodified",
            "mkl_stand_in": "dot_product_mkl := scipy.sparse a @ b (Intel MKL / sparse_dot_mkl not installed)"}
    with open(os.path.join(HERE, "META.json"), "w") as f:
        json.dump(meta, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
