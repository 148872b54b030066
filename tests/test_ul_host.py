"""CPU side of `haphic cluster --ul`: the native UL reader (hh_ul_*) and haphic_b200/ul.py give the contig paths the
reference's parse_ul_alignments gave for the same BAM (tests/golden/ul_*.npz, made through the pure-Python pysam stand-in),
on the adversarial BAM at several supports and on the UL BAM of every whole-run case; the stand-in decodes the fields the
native reader's events imply; whitelist, per-fragment path arrays and the pair list follow from the paths as the
reference's functions use them."""

import json
import logging
import os
import sys

import numpy as np
import pytest

from tests.util import load_golden

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")
RUN_TAGS = ("ctg", "bins", "norm", "gfa_w05", "gfa_w1", "allelic", "concentrated", "quick_view", "no_path", "correct")


def golden_json(g, key):
    return json.loads(bytes(g[key]).decode())


def _args(path, **kw):
    from argparse import Namespace
    d = dict(ul=path, threads=2, min_ul_mapq=30, min_ul_alignment_length=10000, max_distance_to_end=100,
             max_overlap_ratio=0.5, max_gap_len=10000, min_ul_support=2)
    d.update(kw)
    return Namespace(**d)


@pytest.fixture(scope="module")
def adversarial_bam(tmp_path_factory):
    import __graft_entry__ as g
    g.build()
    from haphic_b200 import hicio, synth
    path = str(tmp_path_factory.mktemp("ul") / "adv.bam")
    hicio.write_ul_bam(path, *synth.ul_adversarial())
    return path


def _paths_hashseed0(path, support):
    """ul.parse_ul_alignments in a process with PYTHONHASHSEED=0, as the goldens were made: where a ring ties for its
    lightest edge, the edge that is cut follows the set order of the component's nodes, in the reference and here."""
    import subprocess
    code = ("import json, logging, sys; sys.path.insert(0, {repo!r}); from argparse import Namespace; from haphic_b200 import ul; "
            "a = Namespace(ul={path!r}, threads=2, min_ul_mapq=30, min_ul_alignment_length=10000, max_distance_to_end=100, "
            "max_overlap_ratio=0.5, max_gap_len=10000, min_ul_support={support}); "
            "print(json.dumps(ul.parse_ul_alignments(a, logging.getLogger('t'))))").format(
                repo=os.path.dirname(HERE), path=path, support=support)
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, PYTHONHASHSEED="0"), capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    return json.loads(r.stdout.splitlines()[-1])


@pytest.mark.parametrize("support", [1, 2, 3, 4])
def test_adversarial_paths_match_reference(adversarial_bam, support):
    want = golden_json(load_golden("ul_parse.npz"), "paths_json")[str(support)]
    assert _paths_hashseed0(adversarial_bam, support) == want


@pytest.mark.parametrize("tag", RUN_TAGS)
def test_run_case_paths_match_reference(tmp_path, tag):
    import __graft_entry__ as g
    g.build()
    from haphic_b200 import synth, ul
    gld = load_golden("ul_{}.npz".format(tag))
    nchr, n_contigs, mean_len, n_pairs, seed, ploidy, n_gfa, no_path = [int(x) for x in gld["case"].tolist()]
    synth.ul_case(nchr, n_contigs, mean_len, n_pairs, seed, str(tmp_path), ploidy=ploidy, n_gfa=n_gfa, no_path=bool(no_path))
    want = golden_json(gld, "path_list")
    if golden_json(gld, "argkw").get("correct_nrounds"):
        # --ul with --correct_nrounds: the reference warns and never reads the UL alignments
        assert want == [] and golden_json(gld, "whitelist") == []
        assert "[run] Ultra-long data are not supported now when assembly correction is enabled" in golden_json(gld, "log_lines")
        return
    paths = _paths_hashseed0(str(tmp_path / "ul.bam"), 2)
    assert paths == want
    assert sorted(ul.whitelist(paths)) == golden_json(gld, "whitelist")


def test_stand_in_decodes_the_events_of_the_native_reader(adversarial_bam):
    """Every event's references are those of a primary / supplementary record pair with the same read name that the
    stand-in decodes, and every reference name and length agrees."""
    sys.path.insert(0, GOLDEN)
    import _pysam_ul
    from haphic_b200 import ul
    names, lengths, events = ul.read_ul_events(adversarial_bam, _args(adversarial_bam))
    f = _pysam_ul.AlignmentFile(adversarial_bam, "rb", format_options=[b"filter=!flag.unmap"])
    assert names == f.references and lengths.tolist() == f.lengths
    by_read = {}
    for aln in f:
        by_read.setdefault(aln.query_name, []).append(aln)
    pairs = set()
    for alns in by_read.values():
        prim = [a for a in alns if a.flag in (0, 16)]
        for p in prim:
            for s in alns:
                if s.is_supplementary:
                    pairs.add((p.reference_id, s.reference_id))
    assert len(events)
    for left, right, prim, supp in events.tolist():
        assert (prim, supp) in pairs
        assert {left >> 1, right >> 1} == {prim, supp}


def test_pair_list_and_fragment_arrays_follow_the_paths():
    from haphic_b200 import ul
    paths = [["x_H", "x_T", "y_bin_T", "y_bin_H", "z_H", "z_T"], ["u_T", "u_H", "v_H", "v_T"]]
    assert ul.whitelist(paths) == {"x", "y_bin", "z", "u", "v"}
    names = ["z", "y_bin", "x", "u", "v", "w"]
    ki, kj, slot = ul.table_pairs(paths, names)
    # sorted by contig name: (x_T, y_bin_T) -> slot 3, (y_bin_H, z_H) -> slot 0, (u_H, v_H) -> slot 0
    assert [(names[a], names[b], s) for a, b, s in zip(ki.tolist(), kj.tolist(), slot.tolist())] == [
        ("x", "y_bin", 3), ("y_bin", "z", 0), ("u", "v", 0)]
    # bins: fragments y_bin_bin1, y_bin_bin2 belong to contig 1 ("y_bin")
    parent = np.array([0, 1, 1, 2, 3, 4, 5], np.int32)
    ul_path, ul_parent = ul.fragment_arrays(paths, names, parent)
    assert ul_path.tolist() == [0, 0, 0, 0, 1, 1, -1]
    assert ul_parent.tolist() == parent.tolist()
    # the host version of add_flank_and_full_links_based_on_ul agrees with the per-fragment arrays
    flank = {("z", "y_bin_bin1"): 3, ("y_bin_bin1", "y_bin_bin2"): 5, ("x", "w"): 7, ("u", "v"): 1, ("x", "u"): 2}
    full = {("x", "y_bin"): 4, ("u", "v"): 2, ("x", "z"): 9}
    ul.add_flank_and_full_links_based_on_ul(paths, flank, full, {"y_bin_bin1", "y_bin_bin2"}, logging.getLogger("t"))
    assert flank == {("z", "y_bin_bin1"): 6, ("y_bin_bin1", "y_bin_bin2"): 5, ("x", "w"): 7, ("u", "v"): 2, ("x", "u"): 2}
    assert full == {("x", "y_bin"): 8, ("u", "v"): 4, ("x", "z"): 9}
    ht = {("x_T", "y_bin_T"): 2, ("u_H", "v_H"): 1}
    ul.add_HT_links_based_on_ul(paths, ht, logging.getLogger("t"))
    assert ht == {("x_T", "y_bin_T"): 4, ("u_H", "v_H"): 2}
