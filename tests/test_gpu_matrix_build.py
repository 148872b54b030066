"""GPU: the matrix build (hh_links_linked_index_phased + hh_matrix_from_links_phased).

The first-seen index, the degrees and the passing count of the flank dict are computed once and reused by the next call
with the same table and the same (keep, hap, w, normalize_by_nlinks); every other call recomputes them.  The column
pointers come from the degrees the index pass counted, and each self loop takes slot 0 of its column.  Every case
compares the index and the canonical CSC with the oracle's dict_to_matrix, or, where the oracle has no restatement
(phasing, normalisation, adopted lists), with a fresh LinkTable that computes everything from scratch."""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from haphic_b200._lib import Context
    c = Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def data():
    from haphic_b200 import synth
    from haphic_b200.links import name_rank
    from oracle import haphic_oracle as orc
    asm = synth.make_assembly(nchr=3, n_contigs=120, mean_len=30000, seed=21)
    pairs = synth.make_pairs(asm, 60000, seed=22).numpy()
    rank = name_rank(asm.names)
    in_nx = np.ones(asm.n, np.uint8)
    ref = orc.count_links_numpy(pairs, asm.lengths, rank, in_nx, 500000)
    hap = (np.arange(asm.n) % 2).astype(np.int32)
    return dict(asm=asm, pairs=pairs, rank=rank, in_nx=in_nx, ref=ref, hap=hap)


def new_table(ctx, d, pairs=None, in_nx=None):
    from haphic_b200.links import LinkTable
    tab = LinkTable(ctx, d["asm"].lengths, d["rank"], d["in_nx"] if in_nx is None else in_nx, 500000)
    tab.add(d["pairs"] if pairs is None else pairs)
    tab.finish()
    return tab


def tail_of(index, keep):
    return np.nonzero((index < 0) & (np.asarray(keep) != 0))[0].astype(np.int32)


def unlinked_tail(flank_keys, keep):
    """kept fragments that no flank entry between kept fragments touches, ascending"""
    keep = np.asarray(keep) != 0
    k = np.asarray(flank_keys, dtype=np.int64).reshape(-1, 2)
    k = k[keep[k[:, 0]] & keep[k[:, 1]]]
    linked = np.zeros(len(keep), bool)
    linked[k.ravel()] = True
    return np.nonzero(keep & ~linked)[0].astype(np.int32)


def oracle(d, keep, add_self_loops=True):
    from oracle import haphic_oracle as orc
    tail = unlinked_tail(d["ref"]["flank_keys"], keep)
    m, index = orc.dict_to_matrix(d["ref"]["flank_keys"], d["ref"]["flank_vals"], keep, tail_order=tail,
                                  add_self_loops=add_self_loops)
    return m, index, tail


def same_csc(a, b):
    assert a.shape == b.shape
    assert np.array_equal(a.indptr, b.indptr)
    assert np.array_equal(a.indices, b.indices)
    assert np.array_equal(a.data.astype(np.float32), b.data.astype(np.float32))


def check_oracle(tab, d, keep, mat, add_self_loops=True):
    m, index, tail = oracle(d, keep, add_self_loops)
    same_csc(mat.to_scipy(), m)
    got, n_linked = tab.linked_index(keep)
    assert np.array_equal(np.where(got >= 0, got, index), index) and n_linked == m.shape[0] - len(tail)


def keep_b(d):
    keep = np.ones(d["asm"].n, np.uint8)
    keep[3::5] = 0
    return keep


# ---- reuse and recompute ------------------------------------------------------------------------

def test_index_then_matrix_same_keep(ctx, data):
    tab = new_table(ctx, data)
    keep = np.ones(data["asm"].n, np.uint8)
    index, _ = tab.linked_index(keep)
    mat = tab.to_matrix(keep, tail_of(index, keep))
    check_oracle(tab, data, keep, mat)
    mat2 = tab.to_matrix(keep, tail_of(index, keep))      # a second matrix from the reused index
    check_oracle(tab, data, keep, mat2)
    mat.close(), mat2.close(), tab.close()


def test_index_then_matrix_other_keep(ctx, data):
    tab = new_table(ctx, data)
    keep = np.ones(data["asm"].n, np.uint8)
    tab.linked_index(keep)
    kb = keep_b(data)
    _, _, tail = oracle(data, kb)
    mat = tab.to_matrix(kb, tail)
    check_oracle(tab, data, kb, mat)
    mat.close(), tab.close()


def test_keep_mutated_in_place(ctx, data):
    tab = new_table(ctx, data)
    keep = np.ones(data["asm"].n, np.uint8)
    tab.linked_index(keep)
    keep[::4] = 0
    _, _, tail = oracle(data, keep)
    mat = tab.to_matrix(keep, tail)
    check_oracle(tab, data, keep, mat)
    mat.close(), tab.close()


def test_matrix_without_prior_index(ctx, data):
    tab = new_table(ctx, data)
    kb = keep_b(data)
    _, _, tail = oracle(data, kb)
    mat = tab.to_matrix(kb, tail)
    check_oracle(tab, data, kb, mat)
    mat.close(), tab.close()


def test_matrix_after_fetch(ctx, data):
    tab = new_table(ctx, data)
    keep = np.ones(data["asm"].n, np.uint8)
    index, _ = tab.linked_index(keep)
    tab.fetch()
    mat = tab.to_matrix(keep, tail_of(index, keep))
    check_oracle(tab, data, keep, mat)
    mat.close(), tab.close()


VARIANTS = [dict(), dict(hap="hap", phasing_weight=0.25), dict(hap="hap2", phasing_weight=0.25),
            dict(hap="hap", phasing_weight=1.0), dict(normalize_by_nlinks=True),
            dict(hap="hap", phasing_weight=0.5, normalize_by_nlinks=True)]


def _args(d, v):
    v = dict(v)
    if "hap" in v:
        v["hap"] = d["hap"] if v["hap"] == "hap" else (d["hap"] ^ (np.arange(d["asm"].n) % 3 == 0)).astype(np.int32)
    return v


def fresh(ctx, d, keep, v, pairs=None, adopt=None):
    """index, tail and canonical CSC of a table that has computed nothing yet"""
    tab = new_table(ctx, d, pairs)
    if adopt is not None:
        tab.adopt(*adopt)
    index, _ = tab.linked_index(keep, **_args(d, v))
    tail = tail_of(index, keep)
    mat = tab.to_matrix(keep, tail, **_args(d, v))
    m = mat.to_scipy()
    mat.close(), tab.close()
    return index, tail, m


@pytest.mark.parametrize("first", range(len(VARIANTS)))
@pytest.mark.parametrize("second", range(len(VARIANTS)))
def test_variant_switch(ctx, data, first, second):
    """linked_index with one (hap, w, normalize) and to_matrix with another: the second is what counts"""
    keep = np.ones(data["asm"].n, np.uint8)
    index, tail, m = fresh(ctx, data, keep, VARIANTS[second])
    tab = new_table(ctx, data)
    tab.linked_index(keep, **_args(data, VARIANTS[first]))
    mat = tab.to_matrix(keep, tail, **_args(data, VARIANTS[second]))
    same_csc(mat.to_scipy(), m)
    got, _ = tab.linked_index(keep, **_args(data, VARIANTS[second]))
    assert np.array_equal(got, index)
    mat.close(), tab.close()


def test_adopt_invalidates_the_index(ctx, data):
    tab = new_table(ctx, data)
    keep = np.ones(data["asm"].n, np.uint8)
    tab.linked_index(keep)
    ent, tot, n_records, n_used = tab.export()
    half = ent[: ent.shape[0] // 2].clone()
    adopt = (half, tot, n_records, n_used, len(data["pairs"]))
    index, tail, m = fresh(ctx, data, keep, {}, adopt=adopt)
    tab.adopt(*adopt)
    mat = tab.to_matrix(keep, tail)
    same_csc(mat.to_scipy(), m)
    got, _ = tab.linked_index(keep)
    assert np.array_equal(got, index)
    mat.close(), tab.close()


# ---- shapes ---------------------------------------------------------------------------------------

def hand_table(ctx, links, n, in_nx=None):
    """a table of n contigs (names in id order) from a list of (a, b) links, each one flank record"""
    from haphic_b200.links import LinkTable
    lengths = np.full(n, 10000, np.int64)
    rank = np.arange(n, dtype=np.int32)
    rec = np.array([[a, 10, b, 20] for a, b in links], np.int32).reshape(-1, 4)
    tab = LinkTable(ctx, lengths, rank, np.ones(n, np.uint8) if in_nx is None else in_nx, 500000)
    if len(rec):
        tab.add(rec)
    tab.finish()
    return tab, rec, lengths, rank


def hand_oracle(rec, lengths, rank, in_nx, keep, add_self_loops=True):
    from oracle import haphic_oracle as orc
    ref = orc.count_links_numpy(rec, lengths, rank, in_nx, 500000)
    tail = unlinked_tail(ref["flank_keys"], keep)
    m, index = orc.dict_to_matrix(ref["flank_keys"], ref["flank_vals"], keep, tail_order=tail, add_self_loops=add_self_loops)
    return m, index, tail


def check_hand(ctx, links, n, keep=None, add_self_loops=True, in_nx=None):
    tab, rec, lengths, rank = hand_table(ctx, links, n, in_nx)
    keep = np.ones(n, np.uint8) if keep is None else keep
    m, index, tail = hand_oracle(rec, lengths, rank, np.ones(n, np.uint8) if in_nx is None else in_nx, keep, add_self_loops)
    got, _ = tab.linked_index(keep)
    assert np.array_equal(np.where(got >= 0, got, index), index)
    mat = tab.to_matrix(keep, tail, add_self_loops=add_self_loops)
    same_csc(mat.to_scipy(), m)
    assert mat.nnz == m.nnz
    mat.close(), tab.close()


@pytest.mark.parametrize("hub", [126, 127, 128, 129, 255, 256, 257])
def test_column_boundaries_around_a_hub(ctx, hub):
    """contig 0 linked to 1..hub first: its column (hub + 1 entries with the self loop) ends just before, at and past
    128 / 256 entries; further links between the leaves fill the following columns"""
    links = [(0, k) for k in range(1, hub + 1)] + [(k, k + 1) for k in range(1, hub, 3)]
    check_hand(ctx, links, hub + 40)
    check_hand(ctx, links, hub + 40, add_self_loops=False)


def test_hub_column_links_every_fragment(ctx):
    n = 700
    links = [(0, k) for k in range(1, n)] + [(k, k + 7) for k in range(1, n - 7, 2)]
    check_hand(ctx, links, n)


def test_many_columns_in_one_stretch(ctx):
    """thousands of columns of two entries (one without self loops)"""
    n = 9000
    links = [(k, k + 1) for k in range(0, n - 1, 2)]
    check_hand(ctx, links, n)
    check_hand(ctx, links, n, add_self_loops=False)


def test_tail_columns_hold_only_their_self_loop(ctx):
    n = 300
    links = [(k, (k * 7 + 3) % 150) for k in range(150) if k != (k * 7 + 3) % 150]
    keep = np.ones(n, np.uint8)
    keep[200:220] = 0
    check_hand(ctx, links, n, keep)


def test_single_fragment(ctx):
    check_hand(ctx, [], 1)
    check_hand(ctx, [(0, 1)], 2, keep=np.array([1, 0], np.uint8))


def test_no_flank_entries(ctx):
    n = 50
    links = [(k, k + 1) for k in range(n - 1)]
    check_hand(ctx, links, n, in_nx=np.zeros(n, np.uint8))
    check_hand(ctx, links, n, in_nx=np.zeros(n, np.uint8), add_self_loops=False)


def test_without_self_loops(ctx, data):
    tab = new_table(ctx, data)
    kb = keep_b(data)
    m, _, tail = oracle(data, kb, add_self_loops=False)
    mat = tab.to_matrix(kb, tail, add_self_loops=False)
    same_csc(mat.to_scipy(), m)
    mat.close(), tab.close()


# ---- errors ---------------------------------------------------------------------------------------

def test_bad_tail_and_bad_keep_raise_and_leak_nothing(ctx):
    from haphic_b200._lib import HHError
    n = 40                                     # 0..19 linked, 20..39 kept but unlinked (the tail), 5 dropped
    links = [(k, (k + 3) % 20) for k in range(20)]
    tab, rec, lengths, rank = hand_table(ctx, links, n)
    keep = np.ones(n, np.uint8)
    keep[5] = 0
    m, index, tail = hand_oracle(rec, lengths, rank, np.ones(n, np.uint8), keep)
    assert len(tail) == 20
    linked = int(np.nonzero(index >= 0)[0][0])
    for bad in (np.append(tail, linked), np.append(tail, 5), np.append(tail, n)):
        with pytest.raises(HHError, match="tail lists an id that is dropped, linked, repeated or out of range"):
            tab.to_matrix(keep, bad.astype(np.int32))
    with pytest.raises(HHError, match="tail lists an id that is dropped, linked, repeated or out of range"):
        tab.to_matrix(keep, np.tile(tail, 3))               # longer than the unlinked fragments: refused before sizing
    with pytest.raises(HHError, match="keep mask and tail do not cover the fragment set exactly"):
        tab.to_matrix(keep, tail[1:])
    for _ in range(2):
        mat = tab.to_matrix(keep, tail)
        same_csc(mat.to_scipy(), m)
        got, _ = tab.linked_index(keep)
        assert np.array_equal(np.where(got >= 0, got, index), index)
        mat.close()
    tab.close()
