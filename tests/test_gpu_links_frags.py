"""GPU parity of fragment-mode link counting (hh_links_create_frags / hh_classify_frag: contigs longer than bin_size split
into bins, parse_alignments 1658-1752), every field of the table bit-exact against oracle.count_frag_links_c -- the
records mapped into fragment space (frag_records) and counted by the C restatement of the counting loop:

  a. the edges layout of tests/frag_edges.py (names whose order flips once '_binK' is appended, 13 bins, a contig exactly
     one bin long, one a bin + 1 bp long, one exactly 3 bins long, positions on bin edges, partial Nx) streamed in
     1-record, uneven, host (numpy / pinned), device and asynchronous chunks, and the reference's links_bins_edges.npz;
  b. records whose ends share a bin that does not exist are skipped, as the reference skips them; the other records that
     name a missing bin are refused, with their count and one of their stream indices, in any chunk and at any offset;
  c. synthetic streams on two shapes (the benchmark's 50k contigs x 20 kb with 5 kb bins; 2k contigs x 500 kb with
     100 kb bins), 1M records with flank / Nx variants, 64 Mi records, and the full 200M-record stream;
  d. the engine: fragment tables are counted directly whatever HH_LINKS_PARTITION says;
  e. stream offsets across 2^31;
  f. the linked index and the link matrix in fragment space, bit for bit, and normalize_by_nlinks;
  g. export / merge and route / add_routed / finish_partition / adopt against the single fragment table."""

import re
import resource
import time

import numpy as np
import pytest
import torch

from tests import frag_edges as E
from tests.test_gpu_links_partitioned import assert_equals_oracle
from tests.util import load_golden

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from haphic_b200._lib import Context
    c = Context(0)
    yield c
    c.close()


def layout(names, lengths, bin_size, nx_frac=1.0, seed=0):
    """The fragment layout of stat_fragments / cluster.fragment_layout: contigs longer than bin_size become bins."""
    from haphic_b200.links import name_rank
    frag_names, frag_base, frag_len = [], [0], []
    for n, ln in zip(names, np.asarray(lengths).tolist()):
        if ln > bin_size:
            nb = -(-ln // bin_size)
            frag_names += ["{}_bin{}".format(n, k + 1) for k in range(nb)]
            frag_len += [bin_size] * (nb - 1) + [ln - (nb - 1) * bin_size]
        else:
            frag_names.append(n)
            frag_len.append(ln)
        frag_base.append(len(frag_names))
    nf = len(frag_names)
    in_nx = (np.random.default_rng(seed).random(nf) < nx_frac).astype(np.uint8)
    return dict(names=list(names), lengths=np.asarray(lengths, np.int64), ctg_rank=name_rank(list(names)),
                bin_size=int(bin_size), frag_names=frag_names, frag_base=np.array(frag_base, np.int32),
                frag_len=np.array(frag_len, np.int64), frag_rank=name_rank(frag_names), frag_in_nx=in_nx)


@pytest.fixture(scope="module")
def edges():
    g = load_golden("links_bins_edges.npz")
    w = layout(g["names"].tolist(), g["lengths"], int(g["bin_size"]))
    assert w["frag_names"] == g["frag_names"].tolist() and np.array_equal(w["frag_base"], g["frag_base"])
    w["frag_in_nx"] = g["frag_in_nx"]
    w["golden"] = g
    return w


def table(ctx, w, flank_bp, capacity_hint=0):
    from haphic_b200.links import LinkTable
    return LinkTable(ctx, w["frag_len"], w["frag_rank"], w["frag_in_nx"], flank_bp, capacity_hint=capacity_hint,
                     frags=dict(ctg_rank=w["ctg_rank"], frag_base=w["frag_base"], bin_size=w["bin_size"]))


def send(tab, rec, cuts, how, offset=0):
    """rec[cuts[k]:cuts[k+1]] per call, from offset: 'numpy', 'pinned', 'device', 'async' or 'mixed' (alternating)."""
    for k in range(len(cuts) - 1):
        part = np.ascontiguousarray(rec[cuts[k]:cuts[k + 1]])
        h = how if how != "mixed" else ("numpy", "device", "pinned")[k % 3]
        if h == "pinned":
            part = torch.from_numpy(part).pin_memory()
        elif h in ("device", "async"):
            part = torch.from_numpy(part).cuda()
        tab.add(part, stream_offset=offset + cuts[k], asynchronous=h == "async")


def oracle_check(tab, w, pairs, flank_bp, offset=0, cap=None):
    """Every field against count_frag_links_c (assert_equals_oracle on the mapped records).  Returns the oracle."""
    from oracle import haphic_oracle as orc
    info = tab.finish()
    assert info.n_records == len(pairs)
    mapped, n_bad, _ = orc.frag_records(pairs, w["frag_base"], w["bin_size"])
    assert n_bad == 0
    return assert_equals_oracle(tab, info, mapped, w["frag_len"], w["frag_rank"], w["frag_in_nx"], flank_bp, offset=offset,
                                cap=cap)


# ---- a. the edges layout ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("how", ["one_record", "uneven", "numpy", "pinned", "device", "async"])
@pytest.mark.parametrize("flank_bp", [1000, 5000])
def test_edges_stream(ctx, edges, how, flank_bp):
    n = 1500 if how == "one_record" else 60000
    rec = E.stream(n, seed=7 + flank_bp)
    if how == "one_record":
        cuts = list(range(n + 1))
    elif how == "uneven":
        cuts = [0, 1, 2, 33, 1000, 1031, 40000, n]
    else:
        cuts = [0, 17, 20000, n]
    tab = table(ctx, edges, flank_bp, capacity_hint=1 << 12 if how == "async" else 0)
    send(tab, rec, cuts, {"one_record": "mixed", "uneven": "mixed"}.get(how, how))
    oracle_check(tab, edges, rec, flank_bp)
    tab.close()


@pytest.mark.parametrize("flank_kb", [1, 5])
def test_edges_fixture_matches_reference(ctx, edges, flank_kb):
    """links_bins_edges.npz, made by the unmodified reference: flank dict order and values, per-fragment totals."""
    g = edges["golden"]
    tab = table(ctx, edges, flank_kb * 1000)
    send(tab, g["pairs"], [0, 1000, 1001, len(g["pairs"])], "mixed")
    oracle_check(tab, edges, g["pairs"], flank_kb * 1000)
    f = tab.fetch()
    sel = np.nonzero(f["flank"] > 0)[0]
    sel = sel[np.argsort(f["first_flank"][sel], kind="stable")]
    p = "flank{}_".format(flank_kb)
    assert np.array_equal(np.stack([f["key_i"][sel], f["key_j"][sel]], 1), g[p + "keys"])
    assert np.array_equal(f["flank"][sel].astype(np.int64), g[p + "vals"])
    want = np.zeros(len(edges["frag_names"]), np.int64)
    want[g[p + "frag_link_ids"]] = g[p + "frag_link_vals"]
    assert np.array_equal(tab.fetch_ctg(), want)
    tab.close()


# ---- b. skipped versus refused ----------------------------------------------------------------------------------------

def with_records(base, extra, at):
    out = np.concatenate([base[:at], extra, base[at:]]).astype(np.int32)
    return out, np.arange(at, at + len(extra))


@pytest.mark.parametrize("where", ["first_chunk", "later_chunk", "offset"])
def test_equal_missing_bins_are_skipped(ctx, edges, where):
    """Intra-contig records whose two ends fall in the same bin that does not exist (position -1, far past the end) are
    skipped, as the reference skips them (1715) before its frag_len_dict lookup (1723): the table finishes and counts
    the rest exactly."""
    g = edges["golden"]
    skip = g["single_recs"][(g["single_outcome"] == E.SKIPPED)]
    base = E.stream(20000, seed=31)
    rec, _ = with_records(base, skip, 5 if where == "first_chunk" else 15000)
    offset = (1 << 31) + 12345 if where == "offset" else 0
    tab = table(ctx, edges, 5000)
    send(tab, rec, [0, 10000, len(rec)], "mixed", offset=offset)
    oracle_check(tab, edges, rec, 5000, offset=offset)
    tab.close()


@pytest.mark.parametrize("where", ["first_chunk", "later_chunk", "offset"])
def test_other_missing_bins_are_refused(ctx, edges, where):
    """Every record that names a missing bin otherwise -- the reference dies with a KeyError (1723) -- fails finish()
    with the number of such records and the stream index of one of them, in whichever chunk and at whatever offset."""
    from haphic_b200._lib import HHError
    g = edges["golden"]
    bad = g["single_recs"][(g["single_outcome"] == E.RAISES)]
    assert len(bad) >= 6
    base = E.stream(20000, seed=32)
    rec, at = with_records(base, np.repeat(bad, 2, axis=0), 5 if where == "first_chunk" else 15000)
    offset = (1 << 31) - 14000 if where == "offset" else 0
    tab = table(ctx, edges, 5000)
    send(tab, rec, [0, 10000, len(rec)], "mixed", offset=offset)
    with pytest.raises(HHError) as e:
        tab.finish()
    m = re.search(r"(\d+) records have a position outside their contig's bins \(e\.g\. record (\d+) of the stream\)",
                  str(e.value))
    assert m, str(e.value)
    assert int(m.group(1)) == len(at)
    assert int(m.group(2)) in set((at + offset).tolist())
    tab.close()
    for one in bad:                                  # each alone is refused too
        tab = table(ctx, edges, 5000)
        tab.add(np.ascontiguousarray(one[None, :]), stream_offset=offset)
        with pytest.raises(HHError, match=r"1 records .*e\.g\. record {} ".format(offset)):
            tab.finish()
        tab.close()


# ---- c. / d. synthetic streams ----------------------------------------------------------------------------------------

SHAPES = {"bench": dict(nchr=24, n=50000, mean_len=20000, bin_size=5000, seed=12345),
          "wide": dict(nchr=8, n=2000, mean_len=500000, bin_size=100000, seed=77)}


@pytest.fixture(scope="module")
def shapes():
    from haphic_b200 import synth
    out = {}
    for k, s in SHAPES.items():
        asm = synth.make_assembly(s["nchr"], s["n"], s["mean_len"], seed=s["seed"])
        out[k] = (asm, layout(asm.names, asm.lengths, s["bin_size"]))
    nf = len(out["bench"][1]["frag_names"])
    assert 150000 < nf < 300000, nf
    return out


def synth_records(asm, n, seed):
    from haphic_b200 import synth
    return synth.make_pairs_range(asm, 0, n, seed=seed, device="cuda")


@pytest.mark.parametrize("shape", ["bench", "wide"])
@pytest.mark.parametrize("flank_kb,nx_frac", [(500, 1.0), (5, 0.7)])
def test_synthetic_1m(ctx, shapes, shape, flank_kb, nx_frac, monkeypatch):
    """1M records in uneven host and device chunks, no capacity hint (the table grows); some records name contigs
    outside the FASTA."""
    monkeypatch.delenv("HH_LINKS_PARTITION", raising=False)
    asm, w0 = shapes[shape]
    w = dict(w0, frag_in_nx=(np.random.default_rng(3).random(len(w0["frag_names"])) < nx_frac).astype(np.uint8))
    rec = synth_records(asm, 1_000_000, seed=11).cpu().numpy()
    rec[::997, 0] = asm.n + 5
    rec[5::1013, 2] = -1
    tab = table(ctx, w, flank_kb * 1000)
    send(tab, rec, [0, 1, 33, 70001, 400000, 400032, len(rec)], "mixed")
    ref = oracle_check(tab, w, rec, flank_kb * 1000)
    intra = int((rec[:, 0] == rec[:, 2]).sum())
    print("\n{} 1M: {} fragments, {} intra-contig records, nnz {}".format(shape, len(w["frag_names"]), intra,
                                                                         len(ref["full_vals"])))
    tab.close()


@pytest.mark.parametrize("shape,partition", [("bench", None), ("bench", "1"), ("wide", None)])
def test_synthetic_64mi_counted_directly(ctx, shapes, shape, partition, monkeypatch):
    """64 Mi records in one device call -- above the 16 Mi-record / 2048-key thresholds of the partitioned engine, whose
    scatter classifies contig records only: a fragment table stays on the direct engine (agg_info all zero), with
    HH_LINKS_PARTITION=1 too, and counts bit-exactly."""
    if partition is None:
        monkeypatch.delenv("HH_LINKS_PARTITION", raising=False)
    else:
        monkeypatch.setenv("HH_LINKS_PARTITION", partition)
    monkeypatch.delenv("HH_LINKS_NPART_LOG", raising=False)
    asm, w = shapes[shape]
    n = 64 << 20
    rec = synth_records(asm, n, seed=21)
    tab = table(ctx, w, 5000)
    tab.add(rec)
    info = tab.finish()
    assert tab.agg_info() == {"buckets": 0, "smem_buckets": 0, "fallback_buckets": 0}
    assert info.n_records == n
    from oracle import haphic_oracle as orc
    mapped, n_bad, _ = orc.frag_records(rec.cpu().numpy(), w["frag_base"], w["bin_size"])
    assert n_bad == 0
    assert_equals_oracle(tab, info, mapped, w["frag_len"], w["frag_rank"], w["frag_in_nx"], 5000, cap=int(info.nnz_full))
    tab.close()


@pytest.fixture(scope="module")
def full_stream(ctx, shapes):
    """The benchmark's 200M-record stream on the benchmark assembly with 5 kb bins, one device call, no capacity hint."""
    asm, w = shapes["bench"]
    t0 = time.time()
    rec = synth_records(asm, 200_000_000, seed=12346)
    tab = table(ctx, w, 500000)
    tab.add(rec)
    info = tab.finish()
    torch.cuda.synchronize()
    t_dev = time.time() - t0
    from oracle import haphic_oracle as orc
    t1 = time.time()
    host = rec.cpu().numpy()
    del rec
    mapped, n_bad, _ = orc.frag_records(host, w["frag_base"], w["bin_size"])
    del host
    assert n_bad == 0
    ref = assert_equals_oracle(tab, info, mapped, w["frag_len"], w["frag_rank"], w["frag_in_nx"], 500000,
                               cap=int(info.nnz_full))
    print("\nfragment mode, 200M records, {} fragments: device build {:.1f} s, oracle + compare {:.1f} s, peak host RSS "
          "{:.1f} GB, nnz_full {}".format(len(w["frag_names"]), t_dev, time.time() - t1,
                                          resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1e6, int(info.nnz_full)))
    yield dict(tab=tab, info=info, ref=ref, w=w)
    tab.close()


def test_synthetic_200m(full_stream):
    info, tab = full_stream["info"], full_stream["tab"]
    assert info.n_records == 200_000_000
    assert tab.agg_info()["buckets"] == 0
    f = tab.fetch()
    assert int(f["full"].astype(np.int64).sum()) == info.n_used


# ---- e. stream offsets across 2^31 -------------------------------------------------------------------------------------

def test_stream_offsets_across_2_31(ctx, edges):
    """First-seen indices straddling 2^31 -- the pairs of ctg3 first appear at index 2^31 -- and a refused record after 2^31 named by its full index."""
    from haphic_b200._lib import HHError
    rec = E.stream(200000, seed=41)
    offset = (1 << 31) - 100000
    ctg3, ctg1, ghost = E.names().index("ctg3"), E.names().index("ctg1"), len(E.LAYOUT)
    early = rec[:100000]
    early[(early[:, 0] == ctg3) | (early[:, 2] == ctg3), 0] = ghost              # skipped records before 2^31
    rec[100000] = (ctg3, 10, ctg1, 10005)
    tab = table(ctx, edges, 1000)
    send(tab, rec, [0, 99999, 100001, len(rec)], "mixed", offset=offset)
    oracle_check(tab, edges, rec, 1000, offset=offset)
    f = tab.fetch()
    first = f["first_full"].astype(np.int64)
    assert (first < 1 << 31).any() and (first > 1 << 31).any()
    e = int(np.nonzero(first == 1 << 31)[0][0])
    assert {int(f["key_i"][e]), int(f["key_j"][e])} == {edges["frag_base"][ctg3], edges["frag_base"][ctg1] + 1}
    tab.close()
    g = edges["golden"]
    bad = g["single_recs"][(g["single_outcome"] == E.RAISES)][:1]
    rec2, at = with_records(rec, bad, 150000)
    tab = table(ctx, edges, 1000)
    send(tab, rec2, [0, 100000, len(rec2)], "mixed", offset=offset)
    with pytest.raises(HHError, match=r"1 records .*e\.g\. record {} ".format(offset + int(at[0]))):
        tab.finish()
    tab.close()


# ---- f. linked index and matrix in fragment space ---------------------------------------------------------------------

@pytest.mark.parametrize("shape", ["edges", "wide"])
def test_linked_index_and_matrix(ctx, edges, shapes, shape):
    """linked_index and to_matrix with a keep mask that drops some bins, bit for bit against dict_to_matrix of the
    oracle's flank dict (first touch, i before j; unlinked kept fragments after them); normalize_by_nlinks within 1e-6."""
    from oracle import haphic_oracle as orc
    if shape == "edges":
        w, rec, flank_bp = edges, E.stream(300000, seed=51), 5000
    else:
        asm, w = shapes["wide"]
        rec, flank_bp = synth_records(asm, 1_000_000, seed=52).cpu().numpy(), 20000
    tab = table(ctx, w, flank_bp)
    send(tab, rec, [0, 1000, len(rec)], "mixed")
    ref = oracle_check(tab, w, rec, flank_bp)
    nf = len(w["frag_names"])
    keep = (np.arange(nf) % 7 != 3).astype(np.uint8)
    keep[w["frag_base"][1]] = 0                                      # the first bin of the second contig
    index, n_linked = tab.linked_index(keep)
    tail = np.nonzero((index < 0) & (keep > 0))[0].astype(np.int32)
    link, oindex = orc.dict_to_matrix(ref["flank_keys"], ref["flank_vals"], keep, tail_order=tail.tolist())
    assert n_linked == int((oindex >= 0).sum()) - len(tail)
    assert np.array_equal(np.where(index >= 0, index, oindex), oindex) and (index[keep == 0] < 0).all()
    m = tab.to_matrix(keep, tail).to_scipy()
    assert np.array_equal(m.indptr, link.indptr) and np.array_equal(m.indices, link.indices)
    assert np.array_equal(m.data, link.data)
    norm = orc.normalize_by_nlinks(ref["flank_keys"], ref["flank_vals"], ref["ctg_link_total"])
    nlink, _ = orc.dict_to_matrix(ref["flank_keys"], norm, keep, tail_order=tail.tolist())
    mn = tab.to_matrix(keep, tail, normalize_by_nlinks=True).to_scipy()
    assert np.array_equal(mn.indptr, nlink.indptr) and np.array_equal(mn.indices, nlink.indices)
    assert np.allclose(mn.data, nlink.data, rtol=1e-6, atol=0)
    tab.close()


# ---- g. merge and routing ---------------------------------------------------------------------------------------------

def whole_table(tab):
    index_keep = np.ones(tab.n_ctg, np.uint8)
    index, nl = tab.linked_index(index_keep)
    m = tab.to_matrix(index_keep, np.nonzero(index < 0)[0].astype(np.int32)).to_scipy()
    return tab.fetch(), tab.fetch_ctg(), index, nl, m


def test_sharded_merge_equals_single(ctx, shapes):
    asm, w = shapes["wide"]
    rec = synth_records(asm, 600_000, seed=61).cpu().numpy()
    one = table(ctx, w, 20000)
    one.add(rec)
    one.finish()
    want = whole_table(one)
    half = len(rec) // 2 + 7
    a, b = table(ctx, w, 20000), table(ctx, w, 20000)
    b.add(rec[half:], stream_offset=half)
    b.finish()
    ent, tot, nrec, nused = b.export()
    a.add(rec[:half], stream_offset=0)
    a.merge(ent, tot, nrec, nused)
    info = a.finish()
    assert info.n_records == len(rec)
    got = whole_table(a)
    for k in want[0]:
        assert np.array_equal(want[0][k], got[0][k]), k
    assert np.array_equal(want[1], got[1]) and np.array_equal(want[2], got[2]) and want[3] == got[3]
    assert (want[4] != got[4]).nnz == 0
    for t in (one, a, b):
        t.close()


@pytest.mark.parametrize("world", [2, 3])
def test_routed_equals_single(ctx, shapes, world):
    """route -> add_routed -> finish_partition -> export -> adopt on one GPU: intra-contig records are routed (they make
    links between the bins of a contig), ids outside the FASTA are dropped, and the adopted union equals the single
    fragment table, index and matrix included."""
    asm, w = shapes["wide"]
    rec = synth_records(asm, 600_000, seed=62).cpu().numpy()
    rec[::991, 0] = asm.n + 3
    valid = int(((rec[:, [0, 2]] >= 0) & (rec[:, [0, 2]] < asm.n)).all(1).sum())
    assert (rec[:, 0] == rec[:, 2]).sum() > 1000
    one = table(ctx, w, 20000)
    one.add(rec)
    info1 = one.finish()
    want = whole_table(one)
    cuts = np.linspace(0, len(rec), world + 1).astype(int)
    cuts[1] += 7
    tabs = [table(ctx, w, 20000) for _ in range(world)]
    routed, n_routed = [], 0
    for r in range(world):
        shard = torch.from_numpy(np.ascontiguousarray(rec[cuts[r]:cuts[r + 1]])).cuda()
        rec_out, pos_out, counts = tabs[r].route(shard, int(cuts[r]), world)
        n_routed += sum(counts)
        routed.append((rec_out, pos_out, np.concatenate([[0], np.cumsum(counts)])))
    assert n_routed == valid
    parts, tots, n_used = [], [], 0
    for d in range(world):
        for r in range(world):
            rec_out, pos_out, off = routed[r]
            tabs[d].add_routed(rec_out[off[d]:off[d + 1]].contiguous(), pos_out[off[d]:off[d + 1]].contiguous())
        n_used += int(tabs[d].finish_partition().n_used)
        ent, tot, _, _ = tabs[d].export()
        parts.append(ent)
        tots.append(tot)
    whole, tot = torch.cat(parts), torch.stack(tots).sum(0)
    for d in (0, world - 1):
        info = tabs[d].adopt(whole, tot, len(rec), n_used, len(rec))
        assert (info.n_records, info.n_used, info.nnz_full, info.nnz_flank) == \
               (info1.n_records, info1.n_used, info1.nnz_full, info1.nnz_flank)
        got = whole_table(tabs[d])
        assert np.array_equal(want[2], got[2]) and want[3] == got[3]
        assert (want[4] != got[4]).nnz == 0
        for k in want[0]:
            assert np.array_equal(want[0][k], got[0][k]), k
        assert np.array_equal(want[1], got[1])
    for t in tabs + [one]:
        t.close()
