"""GPU: the two-pass placement of the matrix build (hh_k_mat_group, hh_k_mat_chunks, hh_k_mat_place).

The passing entries are staged by column group (C = 256 columns up to 2^20 fragments, 1024 at 2^22), then each chunk of at
most 8192 staged records of one group is sorted by column in shared memory and stored in column runs.  These cases sit on
the edges of that layout: a matrix size around one group, tail-only groups, a column longer than a chunk, a group of
several chunks, the value variants with entries in many groups, and the size limit.  Each compares the canonical CSC bit
for bit with the oracle's dict_to_matrix, or with the host dict_to_matrix of the reference's dict operations."""

import numpy as np
import pytest

from tests.test_gpu_matrix_build import check_hand, hand_oracle, hand_table, same_csc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from haphic_b200._lib import Context
    c = Context(0)
    yield c
    c.close()


def chain_and_random(n, extra, seed):
    """every contig of 0..n-1 linked (a chain), plus `extra` random links, many of them between groups"""
    rng = np.random.default_rng(seed)
    links = [(k, k + 1) for k in range(n - 1)]
    a, b = rng.integers(0, n, extra), rng.integers(0, n, extra)
    return links + [(int(x), int(y)) for x, y in zip(a, b) if x != y]


@pytest.mark.parametrize("n", [255, 256, 257, 768])
def test_matrix_sizes_around_a_group(ctx, n):
    """n = C - 1 (a single group), C, C + 1 and 3 C, every column linked"""
    links = chain_and_random(n, 6 * n, seed=n)
    check_hand(ctx, links, n)
    check_hand(ctx, links, n, add_self_loops=False)


def test_tail_only_groups(ctx):
    """200 linked fragments, then 1000 kept but unlinked ones: groups 1 to 4 hold only self loops (or nothing)"""
    links = chain_and_random(200, 2000, seed=3)
    check_hand(ctx, links, 1200)
    check_hand(ctx, links, 1200, add_self_loops=False)


def test_column_longer_than_a_chunk(ctx):
    """Fragments 0..9215 (36 full groups) are linked in pairs first; then fragment 9216 links to every one of them.  Its
    column is the only linked column of group 36: 9216 half-entries, a first chunk entirely in one column, a second chunk
    continuing the same column."""
    m = 9216
    links = [(2 * k, 2 * k + 1) for k in range(m // 2)] + [(m, k) for k in range(m)]
    check_hand(ctx, links, m + 1)
    check_hand(ctx, links, m + 40, add_self_loops=False)


def test_group_of_several_chunks(ctx):
    """every pair of fragments 0..255 linked: group 0 stages 65,280 half-entries, eight chunks, and each of its columns
    crosses chunk boundaries; a second group of 100 columns follows"""
    links = [(a, b) for a in range(256) for b in range(a + 1, 256)] + [(256 + k, k) for k in range(100)]
    check_hand(ctx, links, 356)


@pytest.mark.parametrize("normalize,w,use_ul", [(True, 0.0, False), (False, 0.5, False), (False, 0.0, True),
                                                (True, 0.5, True)])
def test_value_variants_across_groups(ctx, normalize, w, use_ul):
    """normalize_by_nlinks, the phasing reduction and the UL doubling on a matrix of about 700 columns (three groups),
    against the host dict_to_matrix of the reference's dict operations"""
    import scipy.sparse as sp
    from haphic_b200 import cluster, ul
    from haphic_b200.links import link_dicts
    from tests.test_gpu_gfa import _haplotypes, _same, _table
    from tests.test_gpu_ul import _contig_layout, _synthetic_paths
    table, names = _table(ctx, 700, 50000, 300000, 2500, 0)
    contigs, parent = _contig_layout(names)
    paths = _synthetic_paths(contigs, 11, 60) if use_ul else []
    hap = _haplotypes(names, 13) if w else None
    frag_set = {n for k, n in enumerate(names) if k % 11 != 4}
    full, flank, _ht, totals = link_dicts(table, names)
    if normalize:
        cluster.normalize_by_nlinks(flank, totals)
    if use_ul:
        ul.add_flank_and_full_links_based_on_ul(paths, flank, dict(full), set(), cluster.logger)
    if w:
        cluster.reduce_inter_hap_HiC_links(flank, {n: (int(h), 0) for n, h in zip(names, hap.tolist())}, w)
    want, want_index = cluster.dict_to_matrix(flank, frag_set, dense_matrix=False, add_self_loops=True)
    want = sp.csc_matrix(want)
    want.sort_indices()
    assert want.shape[0] > 512
    mat, got_index = cluster.device_matrix(table, names, frag_set, normalize_by_nlinks=normalize, add_self_loops=True, hap=hap,
                                           phasing_weight=w, ul=ul.fragment_arrays(paths, contigs, parent) if use_ul else None)
    got = mat.to_scipy()
    mat.close()
    got.sort_indices()
    assert list(got_index.items()) == list(want_index.items())
    _same(got, want)
    table.close()


def test_size_limit(ctx):
    """2^22 + 1 fragments are refused before the matrix is sized; 2^22 (1024-column groups, 4096 of them) are built"""
    from haphic_b200._lib import HHError
    n = (1 << 22) + 1
    links = chain_and_random(300, 3000, seed=7) + [(300 + 2 * k, 301 + 2 * k) for k in range(0, 4000, 7)]
    tab, rec, lengths, rank = hand_table(ctx, links, n)
    keep = np.ones(n, np.uint8)
    index, n_linked = tab.linked_index(keep)
    tail = np.nonzero(index < 0)[0].astype(np.int32)
    assert n_linked + len(tail) == n
    with pytest.raises(HHError, match="at most 4194304 are supported"):
        tab.to_matrix(keep, tail)
    keep[n - 1] = 0
    m, oindex, otail = hand_oracle(rec, lengths, rank, np.ones(n, np.uint8), keep)
    mat = tab.to_matrix(keep, otail)
    assert mat.n == 1 << 22
    same_csc(mat.to_scipy(), m)
    mat.close(), tab.close()
