"""CPU tests of the host-side parts of the drop-in module (haphic_b200/cluster.py, hicio.py):
FASTA / fragment statistics, filters, dict_to_matrix, readers and writers, against the golden
fixtures produced by the reference.  PYTHONHASHSEED-dependent orders are not asserted here."""

import argparse
import json
import os

import numpy as np
import pytest

from tests.util import csc_from, load_golden


def build_dicts(g):
    names = g["names"].tolist()
    from collections import defaultdict
    flank = defaultdict(int)
    vals = g["flank_norm_vals"] if "flank_norm_vals" in g.files else g["flank_vals"]
    for (a, b), v in zip(g["flank_keys"].tolist(), vals.tolist()):
        flank[(names[a], names[b])] = v
    ctg_links = defaultdict(int)
    for c, v in zip(g["ctg_link_ids"].tolist(), g["ctg_link_vals"].tolist()):
        ctg_links[names[c]] = v
    return names, flank, ctg_links


@pytest.mark.parametrize("tag,nchr,n_contigs,mean_len,seed", [("a", 3, 60, 40000, 101), ("b", 4, 120, 60000, 202)])
def test_fasta_and_fragment_statistics(tmp_path, tag, nchr, n_contigs, mean_len, seed):
    from haphic_b200 import cluster, synth
    g = load_golden("links_{}.npz".format(tag))
    asm = synth.make_assembly(nchr, n_contigs, mean_len, seed=seed)
    assert asm.names == g["names"].tolist()
    fasta = str(tmp_path / "asm.fa")
    synth.write_fasta(asm, fasta, seed=seed + 3)
    fa = cluster.parse_fasta(fasta)
    assert list(fa.keys()) == asm.names
    assert [fa[n][1] for n in asm.names] == g["lengths"].tolist()
    assert [fa[n][2] for n in asm.names] == g["RE_sites"].tolist()
    assert cluster.determine_int_type(fa) == ("int32", "int32")
    out = cluster.stat_fragments(fa, "GATC", dict(), set(), nchrs=nchr, flank=int(g["flank_kb"]), Nx=int(g["Nx"]), bin_size=0)
    _, bin_set, bin_size, frag_len, nx_set, re_dict, split = out
    assert not bin_set and not split
    assert [re_dict[n] for n in asm.names] == g["RE_site_dict"].tolist()
    assert [int(n in nx_set) for n in asm.names] == g["in_nx"].tolist()


@pytest.mark.parametrize("tag", ["a", "b"])
def test_filter_and_host_dict_to_matrix(tag):
    from haphic_b200 import cluster
    g = load_golden("links_{}.npz".format(tag))
    names, flank, ctg_links = build_dicts(g)
    nx = {n for n, f in zip(names, g["in_nx"].tolist()) if f}
    re_dict = dict(zip(names, g["RE_site_dict"].tolist()))
    kept = cluster.filter_fragments(nx, re_dict, 5, ctg_links, "0.2X", "1.9X", 10, "1.5X", 0, flank, dict(), "1.5X", set())
    assert [int(n in kept) for n in names] == g["filtered"].tolist()
    m, index = cluster.dict_to_matrix(flank, kept, dense_matrix=False, add_self_loops=True)
    ref_index = g["matrix_index"]
    # linked fragments get first-seen indices (the unlinked tail depends on the hash seed)
    n_linked = len({a for k in flank for a in k if k[0] in kept and k[1] in kept})
    assert set(index) == kept
    for n in kept:
        i = ref_index[names.index(n)]
        if 0 <= i < n_linked:
            assert index[n] == i
    if n_linked == len(kept):
        ref = csc_from(g, "link", m.shape[0])
        m.sort_indices()
        assert np.array_equal(m.indices, ref.indices) and np.allclose(m.data, ref.data, rtol=1e-7, atol=0)


def test_check_param_and_inflation_values():
    from haphic_b200 import cluster
    from haphic_b200.mcl import inflation_values
    assert cluster.check_param("--x", "0.2X", {"X", "x"}) == (0.2, "X")
    assert cluster.check_param("--x", "1", {"X", "x"}) == (1.0, "")
    with pytest.raises(RuntimeError):
        cluster.check_param("--x", "1.5", {"X", "x"})
    with pytest.raises(RuntimeError):
        cluster.check_param("--x", "", {"X", "x"})
    assert [str(v) for v in inflation_values(1.1, 3.0, 0.1)][::19] == ["1.1", "3.0"]
    assert [str(v) for v in inflation_values(1.2, 2.0, 0.2)] == ["1.2", "1.4", "1.6", "1.8", "2.0"]
    # numpy.arange over Decimals keeps element 0 as given: '1.0', not '1.00' (directory names inflation_1.0, ...)
    assert [str(v) for v in inflation_values(1.0, 1.5, 0.25)] == ["1.0", "1.25", "1.50"]
    import numpy
    from decimal import Decimal
    assert [str(v) for v in numpy.arange(Decimal("1.0"), Decimal("1.5") + Decimal("0.25"), Decimal("0.25"))] == ["1.0", "1.25", "1.50"]
    assert cluster.parse_RE_sites(["GANTC"]) == ["GAATC", "GATTC", "GACTC", "GAGTC"]
    assert cluster.count_RE_sites("GATCGATCAAGCTT", "GATC,AAGCTT") == 3


def test_parser_matches_reference_flags():
    from haphic_b200 import cluster
    a = cluster.parse_arguments(["asm.fa", "aln.bam", "12"])
    want = dict(aln_format="auto", RE="GATC", quick_view=False, gfa=None, ul=None, correct_nrounds=0, correct_resolution=500,
                median_cov_ratio=0.2, region_len_ratio=0.1, min_region_cutoff=5000, Nx=80, RE_site_cutoff=5,
                density_lower="0.2X", density_upper="1.9X", read_depth_upper="1.5X", topN=10, rank_sum_hard_cutoff=0,
                rank_sum_upper="1.5X", remove_allelic_links=0, concordance_ratio_cutoff=0.2, nwindows=50,
                remove_concentrated_links=False, max_read_pairs=200, min_read_pairs=20, phasing_weight=1.0, min_ul_mapq=30,
                min_ul_alignment_length=10000, max_distance_to_end=100, max_overlap_ratio=0.5, max_gap_len=10000,
                min_ul_support=2, bin_size=-1, flank=500, normalize_by_nlinks=False, expansion=2, min_inflation=1.1,
                max_inflation=3.0, inflation_step=0.1, max_iter=200, pruning=0.0001, skip_clustering=False, threads=8,
                dense_matrix=False, verbose=False, fasta="asm.fa", alignments="aln.bam", nchrs=12)
    assert vars(a) == want


def test_pairs_and_bam_readers_agree(tmp_path):
    from haphic_b200 import hicio, synth
    asm = synth.make_assembly(2, 20, 30000, seed=9)
    pairs = synth.make_pairs(asm, 5000, seed=10).numpy()
    names = asm.names + ["not_in_fasta"]
    pairs[::50, 2] = asm.n              # a reference that the FASTA does not have
    ext = synth.Assembly(names, None, None, None, None, asm.chrom_len, asm.nchr)
    ppath, bpath = str(tmp_path / "a.pairs"), str(tmp_path / "a.bam")
    synth.write_pairs(ext, pairs, ppath)
    hicio.write_bam(bpath, names, asm.lengths.tolist() + [1000], pairs)
    idx = hicio.NameIndex(asm.names)
    want = pairs[pairs[:, 0] != pairs[:, 2]].copy()
    want[:, 0][want[:, 0] == asm.n] = -1
    want[:, 2][want[:, 2] == asm.n] = -1
    got_p = np.concatenate(list(hicio.pairs_batches(ppath, "pairs", idx, bed_path=str(tmp_path / "a.bed"), batch_lines=700)))
    got_b = np.concatenate(list(hicio.bam_batches(bpath, idx, batch_records=333)))
    assert np.array_equal(got_p, want) and np.array_equal(got_b, want)
    with open(tmp_path / "a.bed") as f:
        bed = f.read().splitlines()
    assert len(bed) == 2 * len(pairs)
    a, pa, b, pb = pairs[0].tolist()
    assert bed[0] == "{}\t{}\t{}\tr0/1\t255\t.".format(names[a], pa, pa)
    assert bed[1] == "{}\t{}\t{}\tr0/2\t255\t.".format(names[b], pb, pb)
    # coordinate-sorted BAMs are refused like the reference does
    hicio.write_bam(bpath, names, asm.lengths.tolist() + [1000], pairs[:10], sort_order="coordinate")
    with pytest.raises(RuntimeError):
        list(hicio.bam_batches(bpath, idx))


@pytest.mark.parametrize("threads", [1, 4])
def test_native_bam_reader_matches_python_decoder(tmp_path, threads):
    """hh_bam_* (threaded BGZF inflate + record walk) against an independent gzip/numpy decoder: many BGZF blocks,
    records straddling block and batch boundaries, intra-contig pairs kept when inter_only is off, unmapped mates,
    truncated files."""
    from haphic_b200 import hicio, synth
    from haphic_b200._lib import HHError
    from tests.util import bam_batches_py
    asm = synth.make_assembly(3, 40, 30000, seed=19)
    pairs = synth.make_pairs(asm, 60000, seed=20).numpy()        # ~8 MB of records -> > 100 BGZF blocks
    pairs[::97, 2] = -1                                          # mate unmapped: next_refID = -1
    pairs[5::101, 0] = asm.n                                     # reference missing from the FASTA
    names = asm.names + ["ghost"]
    bpath = str(tmp_path / "big.bam")
    hicio.write_bam(bpath, names, asm.lengths.tolist() + [500], pairs, sort_order="queryname")
    idx = hicio.NameIndex(asm.names)
    for inter_only in (True, False):
        want = np.concatenate(list(bam_batches_py(bpath, idx, inter_only=inter_only, batch_bytes=1 << 20)))
        got = np.concatenate(list(hicio.bam_batches(bpath, idx, inter_only=inter_only, batch_records=7777, threads=threads)))
        assert np.array_equal(got, want)
        sel = np.ones(len(pairs), bool) if not inter_only else pairs[:, 0] != pairs[:, 2]
        assert len(got) == int(sel.sum())
    # a file cut in the middle of a block / of a record is an error, never a silent short read
    raw = open(bpath, "rb").read()
    cut = str(tmp_path / "cut.bam")
    with open(cut, "wb") as f:
        f.write(raw[: len(raw) // 2])
    with pytest.raises(HHError):
        list(hicio.bam_batches(cut, idx, threads=threads))
    with open(cut, "wb") as f:
        f.write(b"not a bam at all" * 10)
    with pytest.raises(HHError):
        list(hicio.bam_batches(cut, idx, threads=threads))


def test_clm_writer_matches_reference(tmp_path, monkeypatch):
    from haphic_b200 import cluster
    from haphic_b200.links import name_rank
    g = load_golden("links_a.npz")
    names = g["names"].tolist()
    rec = g["pairs"]
    n = len(names)
    ok = (rec[:, 0] != rec[:, 2]) & (rec[:, 0] < n) & (rec[:, 2] < n)
    clm = cluster.build_clm_dict(rec[ok], names, g["lengths"], name_rank(names))
    keys = [[names.index(a), names.index(b)] for a, b in clm.keys()]
    assert keys == g["clm_keys"].tolist()
    assert sum((list(v) for v in clm.values()), []) == g["clm_vals"].tolist()
    monkeypatch.chdir(tmp_path)
    cluster.output_clm(clm)
    with open("paired_links.clm") as f:
        assert f.read() == str(g["clm_text"])


def test_native_clm_writer_matches_reference(tmp_path):
    from haphic_b200 import cluster
    from haphic_b200.links import name_rank
    g = load_golden("links_a.npz")
    names = g["names"].tolist()
    rec = g["pairs"]
    n = len(names)
    ok = (rec[:, 0] != rec[:, 2]) & (rec[:, 0] < n) & (rec[:, 2] < n)
    out = str(tmp_path / "paired_links.clm")
    cluster.write_clm(rec[ok], names, g["lengths"], name_rank(names), out)
    with open(out) as f:
        assert f.read() == str(g["clm_text"])


def test_native_pairs_reader_gz_and_comments(tmp_path):
    import gzip
    from haphic_b200 import hicio
    names = ["ctgA", "ctgB", "c"]
    text = ("## pairs format v1.0\n#columns: readID chr1 pos1 chr2 pos2 strand1 strand2\n"
            "r1\tctgA\t10\tctgB\t20\t+\t-\n\n   \n"
            "r2 ctgB  5   ctgB 9 + +\n"
            "r3\tnope\t7\tc\t1\t-\t-\n"
            "r4\tc\t3\tctgA\t4")                      # last line without newline
    p = tmp_path / "a.pairs.gz"
    with gzip.open(p, "wt") as f:
        f.write(text)
    idx = hicio.NameIndex(names)
    got = np.concatenate(list(hicio.pairs_batches(str(p), "bgzipped_pairs", idx, bed_path=str(tmp_path / "a.bed"), batch_lines=2)))
    assert got.tolist() == [[0, 9, 1, 19], [-1, 6, 2, 0], [2, 2, 0, 3]]
    bed = (tmp_path / "a.bed").read_text().splitlines()
    assert bed == ["ctgA\t9\t9\tr1/1\t255\t.", "ctgB\t19\t19\tr1/2\t255\t.", "ctgB\t4\t4\tr2/1\t255\t.", "ctgB\t8\t8\tr2/2\t255\t.",
                   "nope\t6\t6\tr3/1\t255\t.", "c\t0\t0\tr3/2\t255\t.", "c\t2\t2\tr4/1\t255\t.", "ctgA\t3\t3\tr4/2\t255\t."]
    all_pairs = np.concatenate(list(hicio.pairs_batches(str(p), "bgzipped_pairs", idx, bed_path=None, inter_only=False)))
    assert all_pairs.tolist() == [[0, 9, 1, 19], [1, 4, 1, 8], [-1, 6, 2, 0], [2, 2, 0, 3]]


@pytest.mark.parametrize("compress", ["plain", "gzip", "bgzf"])
@pytest.mark.parametrize("threads", [1, 5])
def test_native_pairs_reader_threads_and_compressions(tmp_path, compress, threads):
    """The threaded tokenizer gives the same records and the same alignments.bed whatever the thread count, the
    compression (plain text, one gzip stream, blocked gzip inflated in parallel) and the batch size; malformed lines
    are reported with their line number."""
    import gzip
    from haphic_b200 import hicio, synth
    from haphic_b200._lib import HHError
    asm = synth.make_assembly(3, 300, 30000, seed=31)
    pairs = synth.make_pairs(asm, 120000, seed=32).numpy()        # ~6 MB of text: several slices per window
    names = asm.names
    lines = ["## pairs format v1.0", "#columns: readID chr1 pos1 chr2 pos2 strand1 strand2"]
    lines += ["r{}\t{}\t{}\t{}\t{}\t+\t-".format(k, names[a], pa + 1, names[b], pb + 1) for k, (a, pa, b, pb) in enumerate(pairs.tolist())]
    text = ("\n".join(lines) + "\n").encode()
    path = str(tmp_path / ("a.pairs" if compress == "plain" else "a.pairs.gz"))
    with open(path, "wb") as f:
        if compress == "plain":
            f.write(text)
        elif compress == "gzip":
            f.write(gzip.compress(text, 1))
        else:
            for i in range(0, len(text), 0xFF00):
                f.write(hicio._bgzf_block(text[i:i + 0xFF00]))
            f.write(hicio._bgzf_block(b""))
    fmt = "pairs" if compress == "plain" else "bgzipped_pairs"
    idx = hicio.NameIndex(names)
    bed = str(tmp_path / "a.bed")
    got = np.concatenate(list(hicio.pairs_batches(path, fmt, idx, bed_path=bed, batch_lines=9999, threads=threads)))
    assert np.array_equal(got, pairs[pairs[:, 0] != pairs[:, 2]])
    want_bed = "".join("{}\t{}\t{}\tr{}/1\t255\t.\n{}\t{}\t{}\tr{}/2\t255\t.\n".format(names[a], pa, pa, k, names[b], pb, pb, k)
                       for k, (a, pa, b, pb) in enumerate(pairs.tolist()))
    with open(bed) as f:
        assert f.read() == want_bed
    if compress == "plain":
        bad = lines[:50002] + ["r\tx\tnotanumber\ty\t5"] + lines[50002:]
        with open(path, "w") as f:
            f.write("\n".join(bad) + "\n")
        with pytest.raises(HHError, match="line 50003"):
            list(hicio.pairs_batches(path, fmt, idx, bed_path=None, threads=threads))


@pytest.mark.parametrize("tag", ["p2", "p4", "p4bins"])
def test_allelic_link_removal_matches_reference_golden(tag):
    """record_coord_pairs / concordance + concentration ratios / remove_allelic_HiC_links (HapHiC_cluster.py:419-692)
    against dicts frozen from the unmodified reference (tests/golden/make_golden.py allelic_case)."""
    import logging
    from math import ceil
    from haphic_b200 import allelic, cluster
    from haphic_b200.links import name_rank
    g = load_golden("allelic_{}.npz".format(tag))
    names = g["names"].tolist()
    lengths = g["lengths"].astype(np.int64)
    kw = json.loads(str(g["argkw"]))
    args = argparse.Namespace(remove_allelic_links=kw["remove_allelic_links"], remove_concentrated_links=kw["remove_concentrated_links"],
                              max_read_pairs=kw.get("max_read_pairs", 200), min_read_pairs=20, nwindows=50,
                              concordance_ratio_cutoff=0.2)
    rank = name_rank(names)
    pairs = g["pairs"]
    rec = pairs[pairs[:, 0] != pairs[:, 2]]
    coord = allelic.coord_pair_dict(rec, names, lengths, rank, args)
    want = json.loads(str(g["coord_json"]))
    assert [list(k) for k in coord.keys()] == [w[:2] for w in want]            # first-seen order of the contig pairs
    n_ratio = 0
    for (key, data), w in zip(coord.items(), want):
        if w[2] is not None:
            assert isinstance(data, list) and data == w[2], key               # [concordance, adj] bit-identical floats
            n_ratio += 1
        else:
            assert not isinstance(data, list) and data.tolist() == w[3], key
    assert n_ratio > 50
    fa_dict = {n: [None, int(l), 0] for n, l in zip(names, lengths)}
    c2f = None
    if "c2f_json" in g:
        bin_size = int(g["bin_size"])
        frag_names, frag_base = [], [0]
        for n, l in zip(names, lengths.tolist()):
            frag_names += ["{}_bin{}".format(n, k + 1) for k in range(ceil(l / bin_size))] if l > bin_size else [n]
            frag_base.append(len(frag_names))
        c2f = allelic.ctg_pair_to_frag_dict(rec, names, rank, frag_names, frag_base, name_rank(frag_names), bin_size)
        got = sorted([[a, b, sorted(map(list, v))] for (a, b), v in c2f.items()])
        assert got == json.loads(str(g["c2f_json"]))
    full = {(a, b): v for a, b, v in json.loads(str(g["full_before_json"]))}
    flank = {(a, b): v for a, b, v in json.loads(str(g["flank_before_json"]))}
    filtered = set(json.loads(str(g["filtered_json"])))
    remaining = cluster.remove_allelic_HiC_links(fa_dict, coord, full, args, flank, filtered, c2f, logger=logging.getLogger("t"))
    assert [[a, b, v] for (a, b), v in full.items()] == json.loads(str(g["full_after_json"]))
    assert [[a, b, v] for (a, b), v in flank.items()] == json.loads(str(g["flank_after_json"]))
    assert sorted(remaining) == json.loads(str(g["remaining_json"]))
    assert len(full) < len(json.loads(str(g["full_before_json"]))) // 2            # the case really removes links
    # run() leaves out the pairs below --min_read_pairs (they only get a debug line): same removals
    sparse = allelic.coord_pair_dict(rec, names, lengths, rank, args, skip_below=args.min_read_pairs)
    assert len(sparse) < len(coord) and all(k in coord for k in sparse)
    full2 = {(a, b): v for a, b, v in json.loads(str(g["full_before_json"]))}
    flank2 = {(a, b): v for a, b, v in json.loads(str(g["flank_before_json"]))}
    remaining2 = cluster.remove_allelic_HiC_links(fa_dict, sparse, full2, args, flank2, set(json.loads(str(g["filtered_json"]))), c2f,
                                                  logger=logging.getLogger("t"))
    assert list(full2.items()) == list(full.items()) and list(flank2.items()) == list(flank.items()) and remaining2 == remaining


def test_array_backed_links_give_the_same_pickles(tmp_path, monkeypatch):
    """run() keeps full_link_dict as arrays (LinkArrays): the native pickles load as the reference's defaultdicts."""
    import pickle
    from haphic_b200 import cluster
    g = load_golden("links_b.npz")
    names = g["names"].tolist()
    rng = np.random.default_rng(4)
    ki, kj = g["full_keys"][:, 0], g["full_keys"][:, 1]
    la = cluster.LinkArrays(names, ki, kj, g["full_vals"])
    full = la.to_dict()
    monkeypatch.chdir(tmp_path)
    la.write_pickle("full_links.pkl")
    with open("full_links.pkl", "rb") as f:
        got = pickle.load(f)
    assert type(got).__name__ == "defaultdict" and got.default_factory is int
    assert got == full and list(got) == list(full)
    ht = rng.integers(0, 3, size=(len(ki), 4)).astype(np.uint32)
    la.write_pickle("HT_links.pkl", ht=ht)
    with open("HT_links.pkl", "rb") as f:
        got = pickle.load(f)
    want = {}
    for e, (a, b) in enumerate(zip(ki.tolist(), kj.tolist())):
        for c in range(4):
            if ht[e, c]:
                want[(names[a] + "_" + "HT"[c >> 1], names[b] + "_" + "HT"[c & 1])] = int(ht[e, c])
    assert got == want


def _python_pairs_reference(text, names, inter_only):
    """pairs_generator / pairs_generator_inter_ctgs (HapHiC_cluster.py:1539-1583) restated literally in Python:
    str.split(), int(), skip blank and '#' lines, BED lines for every data line, `ref != mref` filter."""
    ids = {n: i for i, n in enumerate(names)}
    rec, bed = [], []
    for line in text.split("\n"):
        if not line.strip() or line.startswith("#"):
            continue
        cols = line.split()
        ref, pos, mref, mpos = cols[1], int(cols[2]) - 1, cols[3], int(cols[4]) - 1
        bed.append("{0}\t{1}\t{1}\t{2}/1\t255\t.\n{3}\t{4}\t{4}\t{2}/2\t255\t.\n".format(ref, pos, cols[0], mref, mpos))
        if inter_only and ref == mref:
            continue
        rec.append((ids.get(ref, -1), pos, ids.get(mref, -1), mpos))
    return np.array(rec, dtype=np.int64).reshape(-1, 4), "".join(bed)


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_native_pairs_tokenizer_fuzz_against_python_semantics(tmp_path, seed):
    """Randomly formatted .pairs text (mixed blanks, CRLF, comment and blank lines in the middle, signs / underscores /
    leading zeros in the integers, extra columns, unknown and repeated contig names, missing final newline) must give
    the records and the BED text that Python's str.split() / int() give."""
    import random
    from haphic_b200 import hicio
    rnd = random.Random(seed)
    names = ["ctg{}".format(k) for k in range(40)] + ["scaffold_1|arrow", "x", "chr1_bin2", "A" * 60]
    pool = names + ["unknown_ctg", "ctg1x", "ctg"]

    def blank():
        return rnd.choice([" ", "\t", "  ", "\t\t", " \t", "\x0b", "\x0c"])

    def integer():
        v = rnd.randrange(1, 2_000_000)
        return rnd.choice(["{}", "+{}", "0{}", "{:_}", "00{}"]).format(v)

    lines = ["## pairs format v1.0", "#columns: readID chr1 pos1 chr2 pos2 strand1 strand2"]
    for k in range(30000):
        roll = rnd.random()
        if roll < 0.02:
            lines.append(rnd.choice(["", "   ", "\t", "# a comment", "#"]))
            continue
        a = rnd.choice(pool)
        b = a if rnd.random() < 0.2 else rnd.choice(pool)
        cols = ["read{}".format(k), a, integer(), b, integer()] + ["+", "-", "extra"][: rnd.randrange(0, 4)]
        line = (blank() if rnd.random() < 0.1 else "") + "".join(c + blank() for c in cols[:-1]) + cols[-1]
        lines.append(line + ("\r" if rnd.random() < 0.1 else "") + (blank() if rnd.random() < 0.1 else ""))
    text = "\n".join(lines) + ("" if seed == 2 else "\n")
    path = tmp_path / "fuzz.pairs"
    path.write_bytes(text.encode())
    idx = hicio.NameIndex(names)
    for inter_only in (True, False):
        want_rec, want_bed = _python_pairs_reference(text, names, inter_only)
        bed = str(tmp_path / "fuzz.bed")
        got = list(hicio.pairs_batches(str(path), "pairs", idx, bed_path=bed, batch_lines=4096, inter_only=inter_only, threads=3))
        got = np.concatenate(got) if got else np.zeros((0, 4), np.int32)
        assert np.array_equal(got.astype(np.int64), want_rec)
        with open(bed) as f:
            assert f.read() == want_bed


def _typed_ranking(ranked):
    return {c: [(g, type(v).__name__, repr(v)) for g, v in lst] for c, lst in ranked.items()}


def test_group_link_ranking_on_arrays_equals_the_dict_walk():
    """The array oracle of the reassignment statistics (tests/stats_oracle.py, which the device is compared against at
    size) ranks every contig's groups as the reference's dict walk does (parse_link_dict, then a stable sort by links
    descending): same groups, same sums with the same int / float types, ties in first-met order.  The arrays come from
    the dict by LinkArrays.from_dict, as output_statistics reads a dict."""
    from haphic_b200 import cluster
    from tests import stats_oracle as so
    rng = np.random.default_rng(3)
    n, m = 1500, 120000
    ki, kj = rng.integers(0, n, m), rng.integers(0, n, m)
    ok = ki < kj
    key = np.unique(ki[ok] * n + kj[ok])
    key = key[rng.permutation(len(key))]
    ki, kj = (key // n).tolist(), (key % n).tolist()
    names = ["ctg{}".format(i) for i in range(n)]
    lab = rng.integers(-1, 25, n)
    lab[:40] = -1                                               # contigs 0..39 are ungrouped ...
    groups = {nm: (int(g) if g >= 0 else "ungrouped") for nm, g in zip(names, lab.tolist())}
    only_ungrouped = [(c, c + 1) for c in range(0, 40, 2)]      # ... and some are linked only to each other
    ints = rng.integers(1, 3, len(ki)).tolist()                 # 1 or 2 links: ties everywhere
    frac = rng.choice([0.5, 0.25, 1.5, 0.1], len(ki)).tolist()
    cases = {
        "ints": ints,
        # reduced inter-haplotype links beside counts
        "mixed": [v if rng.random() < 0.5 else v - v * w for v, w in zip(ints, frac)],
        # --remove_concentrated_links scaling: integral floats (`*= 1.0`) and 0.0 among them
        "scaled": [v * r for v, r in zip(ints, rng.choice([1.0, 0.0, 0.5, 2.0], len(ki)).tolist())],
    }
    for tag, vals in cases.items():
        d = {(names[a], names[b]): 3 if tag == "ints" else 3.0 for a, b in only_ungrouped}
        for a, b, v in zip(ki, kj, vals):
            if a >= 40:                                         # (a < b) contigs 0..39 keep only the links above
                d[(names[a], names[b])] = v
        la = cluster.LinkArrays.from_dict(names, d)
        assert [list(k) + [repr(v)] for k, v in la.to_dict().items()] == [list(k) + [repr(v)] for k, v in d.items()], tag
        assert (la.is_float is None) == (tag == "ints"), tag
        gid, ng = so.group_ids(names, groups)
        got = so.ranked_lists(names, *so.ranked_group_links(la, gid, ng))
        want = so.ranked_from_dict(d, groups)
        assert _typed_ranking(got) == _typed_ranking(want), tag
        assert all(names[a] not in want for a, _b in only_ungrouped)
        if tag == "scaled":
            assert any(v == 0.0 for lst in want.values() for _g, v in lst)
            assert any(isinstance(v, float) and v == int(v) and v for lst in want.values() for _g, v in lst)
