"""The fragment-mode oracle (contigs split into bins, parse_alignments 1658-1752) against the fixtures the unmodified
reference produced (links_bins.npz, links_bins_edges.npz), and its two restatements against each other: the per-record
loop on name strings (count_frag_links_loop) and the mapping into fragment space followed by contig-mode counting
(frag_records + count_links_c / count_links_numpy), which is what the GPU tests compare the device with.  CPU only."""

import json
import math

import numpy as np
import pytest

from oracle import haphic_oracle as orc
from tests import frag_edges as E
from tests.util import load_golden


def rank_of(names):
    from haphic_b200.links import name_rank
    return name_rank(list(names))


def fixture(tag, flank_kb=None):
    """(golden, flank_bp, flank keys, flank vals, frag_link ids, frag_link vals) of one fixture and flank size."""
    g = load_golden("links_{}.npz".format(tag))
    if tag == "bins":
        return g, int(g["flank_kb"]) * 1000, g["flank_keys"], g["flank_vals"], g["frag_link_ids"], g["frag_link_vals"]
    p = "flank{}_".format(flank_kb)
    return g, flank_kb * 1000, g[p + "keys"], g[p + "vals"], g[p + "frag_link_ids"], g[p + "frag_link_vals"]


def run_loop(g, flank_bp, pairs=None):
    frag_names = g["frag_names"].tolist()
    nx = {f for f, m in zip(frag_names, g["frag_in_nx"].tolist()) if m}
    return orc.count_frag_links_loop(g["pairs"] if pairs is None else pairs, g["names"].tolist(), g["lengths"],
                                     int(g["bin_size"]), nx, flank_bp)


def run_mapping(g, flank_bp, pairs=None):
    p = g["pairs"] if pairs is None else pairs
    rank = rank_of(g["frag_names"].tolist())
    ref = orc.count_frag_links_c(p, g["frag_base"], int(g["bin_size"]), g["frag_len"], rank, g["frag_in_nx"], flank_bp)
    ref["numpy"] = orc.count_links_numpy(ref["mapped"], g["frag_len"], rank, g["frag_in_nx"], flank_bp, with_clm=False)
    return ref


def loop_arrays(loop, frag_names):
    """The loop's name-keyed flank dict and per-fragment totals as id arrays in insertion order."""
    fid = {f: i for i, f in enumerate(frag_names)}
    keys = np.array([(fid[a], fid[b]) for a, b in loop["flank"]], np.int32).reshape(-1, 2)
    vals = np.array(list(loop["flank"].values()), np.int64)
    tid = np.array([fid[f] for f in loop["frag_links"]], np.int32)
    tval = np.array(list(loop["frag_links"].values()), np.int64)
    return keys, vals, tid, tval


CASES = [("bins", None), ("bins_edges", 1), ("bins_edges", 5)]


@pytest.mark.parametrize("tag,flank_kb", CASES)
def test_loop_matches_reference_fixture(tag, flank_kb):
    """The per-record loop: flank dict order and values, per-fragment totals in insertion order, contig-level full and
    HT dicts."""
    g, flank_bp, fk, fv, tid, tval = fixture(tag, flank_kb)
    loop = run_loop(g, flank_bp)
    assert loop["raises"] == []
    keys, vals, lid, lval = loop_arrays(loop, g["frag_names"].tolist())
    assert np.array_equal(keys, fk) and np.array_equal(vals, fv)
    assert np.array_equal(lid, tid) and np.array_equal(lval, tval)
    assert list(loop["frag_len"]) == g["frag_names"].tolist()
    assert list(loop["frag_len"].values()) == g["frag_len"].tolist()
    names = g["names"].tolist()
    cid = {n: i for i, n in enumerate(names)}
    assert np.array_equal(np.array([(cid[a], cid[b]) for a, b in loop["full"]], np.int32).reshape(-1, 2), g["full_keys"])
    assert list(loop["full"].values()) == g["full_vals"].tolist()
    hk = [(cid[a[:-2]], int(a.endswith("_T")), cid[b[:-2]], int(b.endswith("_T"))) for a, b in loop["HT"]]
    assert np.array_equal(np.array(hk, np.int32).reshape(-1, 4), g["HT_keys"])
    assert list(loop["HT"].values()) == g["HT_vals"].tolist()


@pytest.mark.parametrize("tag,flank_kb", CASES)
def test_mapping_matches_reference_fixture(tag, flank_kb):
    """frag_records + count_links_c: flank dict order and values, per-fragment totals (and, through count_links_numpy,
    their insertion order); the contig-level full and HT dicts are contig-mode counts of the same records."""
    g, flank_bp, fk, fv, tid, tval = fixture(tag, flank_kb)
    ref = run_mapping(g, flank_bp)
    assert ref["n_refused"] == 0
    assert np.array_equal(ref["flank_keys"], fk) and np.array_equal(ref["flank_vals"], fv)
    want = np.zeros(len(g["frag_names"]), np.int64)
    want[tid] = tval
    assert np.array_equal(ref["ctg_link_total"], want)
    assert np.array_equal(ref["numpy"]["ctg_link_ids"], tid) and np.array_equal(ref["numpy"]["ctg_link_vals"], tval)
    for k in ("full_keys", "full_vals", "flank_keys", "flank_vals"):
        assert np.array_equal(ref[k], ref["numpy"][k]), k
    names = g["names"].tolist()
    ctg = orc.count_links_c(g["pairs"], g["lengths"], rank_of(names), np.zeros(len(names), np.uint8), 0)
    assert np.array_equal(ctg["full_keys"], g["full_keys"]) and np.array_equal(ctg["full_vals"], g["full_vals"])
    got = {(i, c >> 1, j, c & 1): v for (i, j), row in zip(ctg["full_keys"].tolist(), ctg["ht"].tolist())
           for c, v in enumerate(row) if v}
    assert got == {tuple(k): v for k, v in zip(g["HT_keys"].tolist(), g["HT_vals"].tolist())}


def test_edges_fixture_reaches_the_edges():
    """The edges stream holds what it is there for: split x unsplit pairs re-sorted by bin name, keys between bin 10+
    and bin 2..9 of one contig, intra-contig pairs, positions on bin edges, fragments both in and out of Nx."""
    g = load_golden("links_bins_edges.npz")
    frag_names = g["frag_names"].tolist()
    c2f = {(a, b): {tuple(x) for x in v} for a, b, v in json.loads(str(g["c2f_json"]))}
    assert ("ctg10", "ctg1_bin1") in c2f[("ctg1", "ctg10")]                   # contig order and bin order disagree
    assert ("ctg2_bin1", "ctg3") in c2f[("ctg2", "ctg3")]                     # and agree
    assert any(a in ("ctg1_bin{}".format(k) for k in range(10, 14)) and b in ("ctg1_bin{}".format(k) for k in range(2, 10))
               for a, b in c2f[("ctg1", "ctg1")])
    assert ("ctg1A", "ctg1_bin1") in c2f[("ctg1", "ctg1A")]
    assert len(g["flank1_keys"]) < len(g["flank5_keys"])
    p = g["pairs"]
    bs = int(g["bin_size"])
    assert ((p[:, 0] == p[:, 2]) & (p[:, 1] // bs != p[:, 3] // bs)).any()
    assert np.isin(p[:, [1, 3]] % bs, [0, bs - 1]).sum() > len(p) // 10
    assert 0 < g["frag_in_nx"].sum() < len(frag_names)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_loop_and_mapping_agree_on_random_streams(seed):
    """Seeded streams over the edges layout with the refused and skipped single records planted at random places: the
    same flank dict, totals and refused records from both restatements."""
    g = load_golden("links_bins_edges.npz")
    rng = np.random.default_rng(seed)
    base = E.stream(4000, 100 + seed)
    bad = E.single_records()
    at = np.sort(rng.choice(len(base) + len(bad), len(bad), replace=False))
    pairs = np.empty((len(base) + len(bad), 4), np.int32)
    mask = np.zeros(len(pairs), bool)
    mask[at] = True
    pairs[mask] = bad
    pairs[~mask] = base
    for flank_bp in (0, 1000, 5000):
        loop = run_loop(g, flank_bp, pairs)
        ref = run_mapping(g, flank_bp, pairs)
        keys, vals, lid, lval = loop_arrays(loop, g["frag_names"].tolist())
        assert np.array_equal(keys, ref["flank_keys"]) and np.array_equal(vals, ref["flank_vals"])
        assert np.array_equal(lid, ref["numpy"]["ctg_link_ids"]) and np.array_equal(lval, ref["numpy"]["ctg_link_vals"])
        assert loop["raises"] == ref["refused"].tolist()
        assert ref["n_refused"] == int((g["single_outcome"] == E.RAISES).sum())


def test_single_records_get_the_reference_outcome():
    """Each single record: skipped, counted or refused (the reference raises) -- by the loop and by the mapping."""
    g = load_golden("links_bins_edges.npz")
    assert np.array_equal(g["single_recs"], E.single_records())
    rank = rank_of(g["frag_names"].tolist())
    for rec, want in zip(g["single_recs"], g["single_outcome"].tolist()):
        rec = rec[None, :]
        loop = run_loop(g, 0, rec)
        got_loop = E.RAISES if loop["raises"] else (E.COUNTED if loop["ctg_pair_to_frag"] else E.SKIPPED)
        mapped, n_bad, bad = orc.frag_records(rec, g["frag_base"], int(g["bin_size"]))
        if n_bad:
            got_map = E.RAISES
            assert bad.tolist() == [0]
        else:
            got_map = E.COUNTED if orc.count_links_c(mapped, g["frag_len"], rank, g["frag_in_nx"], 0)["n_used"] else E.SKIPPED
        assert got_loop == want and got_map == want, (rec.tolist(), want, got_loop, got_map)


@pytest.mark.parametrize("tag", ["bins", "bins_edges"])
def test_ctg_pair_to_frag_matches_loop(tag):
    """allelic.ctg_pair_to_frag_dict (inter-contig records) against the loop's ctg_pair_to_frag, and for the edges
    fixture against the reference's own dict."""
    from haphic_b200 import allelic
    g, flank_bp = fixture(tag, 5)[:2]
    names, frag_names = g["names"].tolist(), g["frag_names"].tolist()
    p = g["pairs"]
    inter = p[(p[:, 0] != p[:, 2]) & (p[:, [0, 2]] >= 0).all(1) & (p[:, [0, 2]] < len(names)).all(1)]
    got = allelic.ctg_pair_to_frag_dict(inter, names, rank_of(names), frag_names, g["frag_base"], rank_of(frag_names),
                                        int(g["bin_size"]))
    loop = run_loop(g, flank_bp)
    want = {k: v for k, v in loop["ctg_pair_to_frag"].items() if k[0] != k[1]}
    assert dict(got) == want
    if tag == "bins_edges":
        ref = {(a, b): {tuple(x) for x in v} for a, b, v in json.loads(str(g["c2f_json"]))}
        assert {k: v for k, v in ref.items() if k[0] != k[1]} == want
        assert dict(loop["ctg_pair_to_frag"]) == ref


@pytest.mark.parametrize("tag", ["bins", "bins_edges"])
def test_fragment_layout_matches_reference(tag):
    """cluster.stat_fragments + fragment_layout give the reference's fragment names, frag_base, lengths and Nx set:
    contigs exactly bin_size long stay whole, bin_size + 1 gives a 1-bp last bin, exact multiples no empty bin."""
    from haphic_b200 import cluster
    g = load_golden("links_{}.npz".format(tag))
    names, lengths = g["names"].tolist(), g["lengths"].tolist()
    fa_dict = {n: ["A" * ln, ln, 1] for n, ln in zip(names, lengths)}
    bin_kb = int(g["bin_size"]) // 1000
    _, _, bin_size, frag_len_dict, nx_set, _, split = cluster.stat_fragments(fa_dict, "GATC", dict(), set(), nchrs=2,
                                                                             flank=0, Nx=int(g["Nx"]), bin_size=bin_kb)
    assert bin_size == int(g["bin_size"])
    frag_names, frag_base, frag_len, frag_rank, in_nx = cluster.fragment_layout(fa_dict, bin_size, frag_len_dict, nx_set, split)
    assert frag_names == g["frag_names"].tolist()
    assert np.array_equal(frag_base, g["frag_base"]) and np.array_equal(frag_len, g["frag_len"])
    assert np.array_equal(in_nx, g["frag_in_nx"]) and np.array_equal(frag_rank, rank_of(frag_names))
    nb = np.diff(frag_base)
    for ln, k in zip(lengths, nb.tolist()):
        assert k == (1 if ln <= bin_size else math.ceil(ln / bin_size))
    if tag == "bins_edges":
        by = dict(zip(names, nb.tolist()))
        assert (by["ctg1A"], by["ctg1_x"], by["ctg1a"], by["ctg1"]) == (1, 2, 3, 13)
        assert frag_len[frag_base[names.index("ctg1_x")] + 1] == 1
