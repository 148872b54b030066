"""GPU side of `haphic cluster --ul`:
  * whole runs write the files, log lines and typed full_links.pkl / HT_links.pkl items the unmodified reference wrote for
    the same inputs (tests/golden/ul_*.npz), from .pairs and, for two cases, from BAM Hi-C input;
  * the device matrix with ul_path / ul_parent (hh_matrix_from_links_ex) is bit-exact against host dict_to_matrix of the
    dict add_flank_and_full_links_based_on_ul leaves, with contigs and bins, with and without normalisation, phased;
  * all-(-1) path arrays and an empty pair list change nothing;
  * fetch / fetch_phased with a pair list equal the host doubling of the plain fetch, HH intact;
  * a count doubled across 2048 takes the f16 pre-expansion's clip correction and M1 stays in its band;
  * at the C3 shape with 2,000 paths the matrix equals a torch reconstruction from the fetched table;
  * with --verbose the array path logs the reference's UL debug lines."""

import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

from tests.test_gpu_gfa import _haplotypes, _same, _table
from tests.test_ul_host import golden_json
from tests.util import load_golden

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COMPARED_LOGS = ("[parse_ul_alignments]", "[filter_fragments]", "[reduce_inter_hap_HiC_links]", "[recommend_inflation]", "[mcl]",
                 "[run] Ultra-long")

DRIVER = r"""
import sys
sys.path.insert(0, {repo!r})
from haphic_b200 import cluster, synth
gfa = synth.ul_case(*{case!r}, ".", ploidy={ploidy}, n_gfa={n_gfa}, bam={bam!r}, no_path={no_path!r})
argv = ["asm.fa", "aln.bam" if {bam!r} else "aln.pairs", str({nchr})] + {extra!r} + ["--ul", "ul.bam"]
if gfa:
    argv += ["--gfa", ",".join(gfa)]
cluster.run(cluster.parse_arguments(argv), log_file="HapHiC_cluster.log")
"""


def typed_items(d):
    return [list(k) + [repr(v)] for k, v in d.items()]


@pytest.mark.parametrize("tag,bam", [("ctg", False), ("ctg", True), ("bins", False), ("bins", True), ("norm", False),
                                     ("gfa_w05", False), ("gfa_w1", False), ("allelic", False), ("concentrated", False),
                                     ("quick_view", False), ("no_path", False), ("correct", False)])
def test_ul_run_matches_reference(tmp_path, tag, bam):
    g = load_golden("ul_{}.npz".format(tag))
    nchr, n_contigs, mean_len, n_pairs, seed, ploidy, n_gfa, no_path = [int(x) for x in g["case"].tolist()]
    extra = []
    for k, v in golden_json(g, "argkw").items():
        if v is True:
            extra.append("--" + k)
        elif v is not False:
            extra += ["--" + k, str(v)]
    code = DRIVER.format(repo=REPO, case=(nchr, n_contigs, mean_len, n_pairs, seed), ploidy=ploidy, n_gfa=n_gfa, bam=bam,
                         no_path=bool(no_path), nchr=nchr, extra=extra)
    r = subprocess.run([sys.executable, "-c", code], cwd=str(tmp_path), env=dict(os.environ, PYTHONHASHSEED="0"),
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    want = golden_json(g, "files_json")
    got = {}
    for root, _d, files in os.walk(tmp_path):
        for fn in files:
            p = os.path.relpath(os.path.join(root, fn), tmp_path)
            if p.startswith("inflation_") and p.endswith(".txt"):
                got[p] = open(os.path.join(root, fn)).read()
    assert sorted(got) == sorted(want)
    for p in sorted(want):
        assert got[p] == want[p], p
    with open(tmp_path / "HapHiC_cluster.log") as f:
        log = [ln.split("> ", 1)[1] for ln in f.read().splitlines() if "> [" in ln]
    assert [ln for ln in log if ln.startswith(COMPARED_LOGS)] == [
        ln for ln in golden_json(g, "log_lines") if ln.startswith(COMPARED_LOGS)]
    if "full_links_items" in g:
        with open(tmp_path / "full_links.pkl", "rb") as f:
            assert typed_items(pickle.load(f)) == golden_json(g, "full_links_items")
    with open(tmp_path / "HT_links.pkl", "rb") as f:
        got_ht = {tuple(k[:2]): k[2] for k in typed_items(pickle.load(f))}
    # HT_link_dict is looked up, never iterated (HapHiC_sort.py:126-131): keys and typed values, order aside
    assert got_ht == {tuple(k[:2]): k[2] for k in golden_json(g, "HT_links_items")}
    import hashlib
    for p, d in golden_json(g, "digests_json").items():
        if p.endswith(".pkl") or (bam and p == "alignments.bed"):
            continue
        assert hashlib.sha1((tmp_path / p).read_bytes()).hexdigest() == d, p


# ------------------------------------------------------------------------------------------------
# the device matrix against host dict_to_matrix of the UL-doubled dict
# ------------------------------------------------------------------------------------------------

def _synthetic_paths(contigs, seed, n_paths):
    """Paths over disjoint random runs of contigs, in node form (c_H, c_T or c_T, c_H per contig)."""
    rng = np.random.default_rng(seed)
    order = rng.permutation(len(contigs)).tolist()
    paths, k = [], 0
    for _ in range(n_paths):
        m = int(rng.integers(2, 6))
        run = order[k:k + m]
        k += m
        path = []
        for c in run:
            ends = ["_H", "_T"] if rng.random() < 0.5 else ["_T", "_H"]
            path += [contigs[c] + e for e in ends]
        paths.append(path)
    return paths


def _contig_layout(names):
    contigs, parent, ids = [], [], {}
    for n in names:
        c = n.rsplit("_bin", 1)[0] if "_bin" in n else n
        if c not in ids:
            ids[c] = len(contigs)
            contigs.append(c)
        parent.append(ids[c])
    return contigs, np.asarray(parent, np.int32)


@pytest.fixture(scope="module")
def ctx():
    from haphic_b200 import cluster
    return cluster._context()


@pytest.mark.parametrize("bins", [False, True])
@pytest.mark.parametrize("normalize", [False, True])
@pytest.mark.parametrize("w", [0.0, 0.5])
def test_ul_matrix_matches_host_dict_to_matrix(ctx, bins, normalize, w):
    import scipy.sparse as sp
    from haphic_b200 import cluster, ul
    from haphic_b200.links import link_dicts
    table, names = _table(ctx, 60 if bins else 160, 300000 if bins else 50000, 120000, 1900 + bins, 120 if bins else 0)
    contigs, parent = _contig_layout(names)
    paths = _synthetic_paths(contigs, 5 + bins, 8 if bins else 20)
    hap = _haplotypes(names, 9) if w else None
    frag_set = {n for k, n in enumerate(names) if k % 9 != 2}
    full, flank, _ht, totals = link_dicts(table, names)
    if normalize:
        cluster.normalize_by_nlinks(flank, totals)
    bin_set = {n for n in names if n not in contigs}
    ul.add_flank_and_full_links_based_on_ul(paths, flank, dict(full), bin_set, cluster.logger)
    if w:
        cluster.reduce_inter_hap_HiC_links(flank, {n: (int(h), 0) for n, h in zip(names, hap.tolist())}, w)
    want, want_index = cluster.dict_to_matrix(flank, frag_set, dense_matrix=False, add_self_loops=True)
    want = sp.csc_matrix(want)
    want.sort_indices()
    mat, got_index = cluster.device_matrix(table, names, frag_set, normalize_by_nlinks=normalize, add_self_loops=True, hap=hap,
                                           phasing_weight=w, ul=ul.fragment_arrays(paths, contigs, parent))
    got = mat.to_scipy()
    mat.close()
    got.sort_indices()
    assert list(got_index.items()) == list(want_index.items())
    _same(got, want)
    assert np.any(got.data != cluster.device_matrix(table, names, frag_set, normalize_by_nlinks=normalize, hap=hap,
                                                    phasing_weight=w)[0].to_scipy().data) or not paths
    table.close()


def test_ul_noops_change_nothing(ctx):
    from haphic_b200 import cluster
    table, names = _table(ctx, 160, 50000, 120000, 2000, 0)
    frag_set = set(names)
    base, base_index = cluster.device_matrix(table, names, frag_set)
    none = (np.full(len(names), -1, np.int32), np.arange(len(names), dtype=np.int32))
    got, index = cluster.device_matrix(table, names, frag_set, ul=none)
    assert list(index.items()) == list(base_index.items())
    a, b = got.to_scipy(), base.to_scipy()
    a.sort_indices()
    b.sort_indices()
    _same(a, b)
    plain = table.fetch()
    hap = _haplotypes(names, 4)
    plain_phased = table.fetch_phased(hap, 0.5)
    table.set_ul_pairs([], [], [])
    again = table.fetch()
    for k in plain:
        assert np.array_equal(plain[k], again[k]), k
    again_phased = table.fetch_phased(hap, 0.5)
    for k in plain_phased:
        assert np.array_equal(plain_phased[k], again_phased[k]), k
    table.close()


def test_ul_fetches_double_the_listed_pairs(ctx):
    table, names = _table(ctx, 160, 50000, 120000, 2100, 0)
    plain = table.fetch()
    hap = _haplotypes(names, 6)
    plain_phased = table.fetch_phased(hap, 0.5)
    rng = np.random.default_rng(3)
    pick = rng.choice(len(plain["key_i"]), 25, replace=False)
    slots = rng.integers(0, 4, 25).astype(np.int32)
    table.set_ul_pairs(plain["key_i"][pick], plain["key_j"][pick], slots)
    got = table.fetch()
    want_full = plain["full"].astype(np.int64)
    want_full[pick] *= 2
    want_ht = plain["ht"].astype(np.int64)
    want_ht[pick, slots] *= 2
    assert np.array_equal(got["full"], want_full)
    assert np.array_equal(got["ht"], want_ht)
    for k in ("key_i", "key_j", "flank", "first_full", "first_flank"):
        assert np.array_equal(got[k], plain[k]), k
    # HH (slot 0) stays full - HT - TH - TT of the stored counts unless it is the doubled slot itself
    keys = set(zip(plain["key_i"][pick].tolist(), plain["key_j"][pick].tolist()))
    got_phased = table.fetch_phased(hap, 0.5)
    doubled = np.array([(a, b) in keys for a, b in zip(plain_phased["key_i"].tolist(), plain_phased["key_j"].tolist())])
    assert np.array_equal(got_phased["values"], np.where(doubled, 2.0, 1.0) * plain_phased["values"])
    assert np.array_equal(got_phased["is_float"], plain_phased["is_float"])
    table.close()


def test_ul_doubling_crosses_the_f16_clip(ctx, monkeypatch):
    """A flank count in (1024, 2048] doubled above 2048: the pre-expansion must see the doubled matrix value and take the
    f16 encoding's clip correction, which the undoubled matrix does not need; M1 stays in the 2e-6 band of the exact
    product.  The oracle doubles the one dict entry by hand."""
    import scipy.sparse as sp
    from haphic_b200 import cluster, synth
    from haphic_b200.links import link_dicts
    from haphic_b200.mcl import Mcl
    from tests.test_gpu_gemm import exact_m1
    monkeypatch.setenv("HH_GEMM_FMT", "f16")
    asm = synth.make_assembly(4, 40, 30000, seed=2300)
    pairs = synth.make_pairs(asm, 10000, seed=2301).numpy()
    a, b = 0, asm.n - 1                                        # first and last chromosome
    extra = np.array([[a, 1000 + k, b, 2000 + k] for k in range(1500)], np.int32)
    names = list(asm.names)
    table, _ = cluster.count_links([np.concatenate([pairs, extra])], names, asm.lengths, set(names), 500, want_clm=False)
    _full, flank, _ht, _tot = link_dicts(table, names)
    key = (names[a], names[b]) if (names[a], names[b]) in flank else (names[b], names[a])
    assert 1024 < flank[key] <= 2048 and max(flank.values()) <= 2048
    flank[key] *= 2
    want, want_index = cluster.dict_to_matrix(flank, set(names), dense_matrix=False, add_self_loops=True)
    want = sp.csc_matrix(want)
    want.sort_indices()
    path = np.full(len(names), -1, np.int32)
    path[[a, b]] = 0
    mat, index = cluster.device_matrix(table, names, set(names), ul=(path, np.arange(len(names), dtype=np.int32)))
    got = mat.to_scipy()
    got.sort_indices()
    assert list(index.items()) == list(want_index.items())
    _same(got, want)
    assert got.data.max() > 2048
    base, _ = cluster.device_matrix(table, names, set(names))
    mc_base = Mcl(base, preexp="dense")
    assert mc_base.preexp["mode"] == "dense" and mc_base.preexp["clip_ms"] == 0
    mc_base.close()
    mc = Mcl(mat, preexp="dense")
    assert mc.preexp["mode"] == "dense" and mc.preexp["clip_ms"] > 0
    m1 = mc.m1().astype(np.float64)
    exact = exact_m1(got)
    nz = exact != 0
    assert np.array_equal(m1 != 0, nz)
    assert (np.abs(m1[nz] - exact[nz]) / exact[nz]).max() <= 2e-6
    mc.close()
    mat.close()
    base.close()
    table.close()


def test_c3_shape_ul_matrix_against_torch(ctx):
    """50k contigs, 200M pairs, 2,000 paths of five consecutive contigs: the device matrix with the UL arrays against a
    torch reconstruction from the fetched table (flank mask, keep mask, x2 where both ends share a path id, first-seen
    indices by the smallest touch), compared entry by entry in canonical CSC order."""
    import torch
    from haphic_b200 import cluster
    table, names = _table(ctx, 50000, 20000, 200_000_000, 2200, 0, device="cuda")
    dev = torch.device("cuda", ctx.device)
    f = table.fetch()
    ki = torch.from_numpy(f["key_i"].astype(np.int64)).to(dev)
    kj = torch.from_numpy(f["key_j"].astype(np.int64)).to(dev)
    flank = torch.from_numpy(f["flank"].astype(np.int64)).to(dev)
    touch_t = torch.from_numpy(f["first_flank"].astype(np.int64)).to(dev) * 2
    del f
    n = len(names)
    rng = np.random.default_rng(23)
    blocks = rng.choice(n // 5, 2000, replace=False)
    path_np = np.full(n, -1, np.int32)
    for k, blk in enumerate(blocks.tolist()):
        path_np[5 * blk:5 * blk + 5] = k
    keep_np = np.arange(n) % 10 != 4
    frag_set = {nm for nm, k in zip(names, keep_np.tolist()) if k}
    path = torch.from_numpy(path_np.astype(np.int64)).to(dev)
    keep = torch.from_numpy(keep_np).to(dev)
    same = (path[ki] >= 0) & (path[ki] == path[kj])
    x = flank.to(torch.float64)
    x = torch.where(same, 2 * x, x)
    sel = (flank > 0) & keep[ki] & keep[kj]
    assert int((sel & same).sum()) > 1000                      # the doubling is exercised
    big = torch.iinfo(torch.int64).max
    touch = torch.full((n,), big, dtype=torch.int64, device=dev)
    touch.scatter_reduce_(0, ki[sel], touch_t[sel], "amin")
    touch.scatter_reduce_(0, kj[sel], touch_t[sel] + 1, "amin")
    linked = touch < big
    order = torch.argsort(touch[linked], stable=True)
    index = torch.full((n,), -1, dtype=torch.int64, device=dev)
    index[torch.nonzero(linked).squeeze(1)[order]] = torch.arange(int(linked.sum()), device=dev)
    mat, got_index = cluster.device_matrix(table, names, frag_set, ul=(path_np, np.arange(n, dtype=np.int32)))
    idx_np = index.cpu().numpy()
    for c in np.nonzero(idx_np >= 0)[0].tolist():
        assert got_index[names[c]] == idx_np[c]
    fi = torch.from_numpy(np.array([got_index.get(nm, -1) for nm in names], np.int64)).to(dev)
    m = len(frag_set)
    r, c, v = fi[ki[sel]], fi[kj[sel]], x[sel].to(torch.float32)
    diag = torch.arange(m, device=dev)
    want_key = torch.cat([c, r, diag]) * m + torch.cat([r, c, diag])
    want_val = torch.cat([v, v, torch.ones(m, dtype=torch.float32, device=dev)])
    want_key, perm = torch.sort(want_key)
    want_val = want_val[perm]
    got = mat.to_scipy()
    mat.close()
    indptr = torch.from_numpy(got.indptr.astype(np.int64)).to(dev)
    got_key = torch.repeat_interleave(torch.arange(m, device=dev), indptr[1:] - indptr[:-1]) * m + \
        torch.from_numpy(got.indices.astype(np.int64)).to(dev)
    got_val = torch.from_numpy(got.data).to(dev)
    assert torch.equal(got_key, want_key)
    assert torch.equal(got_val.view(torch.int32), want_val.view(torch.int32))
    table.close()


def test_ul_verbose_debug_lines_on_the_array_path(tmp_path):
    """With --verbose the array path (doubling inside the device fetch) logs the reference's add_HT_links_based_on_ul and
    add_flank_and_full_links_based_on_ul debug lines, as the host functions log them for the keys the reference's pickles
    hold."""
    import logging
    from haphic_b200 import ul
    g = load_golden("ul_ctg.npz")
    nchr, n_contigs, mean_len, n_pairs, seed, ploidy, n_gfa, no_path = [int(x) for x in g["case"].tolist()]
    extra = ["--Nx", "100", "--bin_size", "0", "--skip_clustering", "--verbose"]
    code = DRIVER.format(repo=REPO, case=(nchr, n_contigs, mean_len, n_pairs, seed), ploidy=ploidy, n_gfa=n_gfa, bam=False,
                         no_path=False, nchr=nchr, extra=extra)
    r = subprocess.run([sys.executable, "-c", code], cwd=str(tmp_path), env=dict(os.environ, PYTHONHASHSEED="0"),
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    tags = ("[add_HT_links_based_on_ul]", "[add_flank_and_full_links_based_on_ul]")
    with open(tmp_path / "HapHiC_cluster.log") as f:
        got = [ln.split("> ", 1)[1] for ln in f.read().splitlines() if "> [" in ln]
    got = [ln for ln in got if ln.startswith(tags)]
    lines = []

    class Capture(logging.Handler):
        def emit(self, rec):
            lines.append("[{}] {}".format(rec.funcName, rec.getMessage()))

    log = logging.getLogger("test_ul_verbose")
    log.setLevel(logging.DEBUG)
    log.addHandler(Capture())
    paths = golden_json(g, "path_list")
    ht_keys = {tuple(k[:2]) for k in golden_json(g, "HT_links_items")}
    full_keys = {tuple(k[:2]) for k in golden_json(g, "full_links_items")}
    ul.add_HT_links_based_on_ul(paths, ht_keys, log)
    ul.add_flank_and_full_links_based_on_ul(paths, None, full_keys, set(), log)
    assert got == lines and len(lines) >= len(ul.adjacent_pairs(paths))
