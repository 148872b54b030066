"""GPU side of `haphic cluster --gfa`:
  * whole runs write the files, log lines and full_links.pkl items (value types included) the unmodified reference wrote
    for the same inputs (tests/golden/gfa_*.npz), from .pairs and from BAM;
  * the phased device matrix (hh_matrix_from_links_phased) is bit-exact against host dict_to_matrix of the dict that
    reduce_inter_hap_HiC_links leaves, with contigs and with bins, with and without normalisation;
  * at the C2 shape it equals a torch reconstruction from the fetched table;
  * one haplotype or w = 0 gives exactly the unphased matrix;
  * a fractional-w matrix takes the weights encoding of the tensor-core pre-expansion and stays in its 2e-6 band."""

import json
import os
import pickle
import subprocess
import sys
from math import ceil

import numpy as np
import pytest
import scipy.sparse as sp

from tests.test_gfa_host import golden_json
from tests.util import load_golden

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COMPARED_LOGS = ("[parse_gfa]", "[filter_fragments]", "[reduce_inter_hap_HiC_links]", "[recommend_inflation]", "[mcl]")

DRIVER = r"""
import sys
sys.path.insert(0, {repo!r})
from haphic_b200 import cluster, synth
gfa = synth.gfa_case(*{case!r}, ".", bam={bam!r})
argv = ["asm.fa", "aln.bam" if {bam!r} else "aln.pairs", str({nchr})] + {extra!r} + ["--gfa", ",".join(gfa)]
cluster.run(cluster.parse_arguments(argv), log_file="HapHiC_cluster.log")
"""


def typed_items(d):
    return [list(k) + [repr(v)] for k, v in d.items()]


@pytest.mark.parametrize("tag,bam", [("w1", False), ("w05_norm", False), ("w05_norm", True), ("one_x", False),
                                     ("one_frac", False), ("bins", False), ("bins", True), ("allelic", False),
                                     ("correct", False), ("correct_qv", False)])
def test_gfa_run_matches_reference(tmp_path, tag, bam):
    g = load_golden("gfa_{}.npz".format(tag))
    case = [int(x) for x in g["case"].tolist()]
    extra = []
    for k, v in golden_json(g, "argkw").items():
        if v is True:
            extra.append("--" + k)
        elif v is not False:
            extra += ["--" + k, str(v)]
    code = DRIVER.format(repo=REPO, case=tuple(case), bam=bam, nchr=case[0], extra=extra)
    r = subprocess.run([sys.executable, "-c", code], cwd=str(tmp_path), env=dict(os.environ, PYTHONHASHSEED="0"),
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    want = golden_json(g, "files_json")
    got = {}
    for root, _d, files in os.walk(tmp_path):
        for fn in files:
            p = os.path.relpath(os.path.join(root, fn), tmp_path)
            full = os.path.join(root, fn)
            if p.startswith("inflation_") and p.endswith(".txt"):
                got[p] = open(full).read()
            elif p.startswith("corrected_") and p.endswith(".gfa"):
                got[p] = ("link:" + os.path.basename(os.readlink(full))) if os.path.islink(full) else open(full).read()
    assert sorted(got) == sorted(want)
    for p in sorted(want):
        assert got[p] == want[p], p
    with open(tmp_path / "HapHiC_cluster.log") as f:
        log = [ln.split("> ", 1)[1] for ln in f.read().splitlines() if "> [" in ln]
    log = [ln for ln in log if ln.startswith(COMPARED_LOGS)]
    want_log = [ln for ln in golden_json(g, "log_lines") if ln.startswith(COMPARED_LOGS)]
    assert [ln.replace(str(tmp_path) + os.sep, "") for ln in log] == [_strip_dirs(ln) for ln in want_log]
    if "full_links_items" in g:
        with open(tmp_path / "full_links.pkl", "rb") as f:
            assert typed_items(pickle.load(f)) == golden_json(g, "full_links_items")
    import hashlib
    digests = golden_json(g, "digests_json")
    for p, d in digests.items():
        if p.endswith(".pkl") or (bam and p == "alignments.bed"):
            continue
        assert hashlib.sha1((tmp_path / p).read_bytes()).hexdigest() == d, p


def _strip_dirs(line):
    k = line.find("/tmp")
    if k < 0:
        return line
    end = line.find(".gfa", k)
    return line.replace(line[k:line.rfind("/", k, end) + 1], "")


# ------------------------------------------------------------------------------------------------
# the phased device matrix against host dict_to_matrix of the reduced dict
# ------------------------------------------------------------------------------------------------

def _table(ctx, n_contigs, mean_len, n_pairs, seed, bin_kb, device="cpu"):
    """(table, fragment names, contig-level table or None): contigs, or fragments with bins of ``bin_kb`` kb."""
    from argparse import Namespace
    from haphic_b200 import cluster, synth
    asm = synth.make_assembly(4, n_contigs, mean_len, seed=seed)
    pairs = synth.make_pairs(asm, n_pairs, seed=seed + 1, homolog=(2, 0.2), device=device)
    if device == "cpu":
        pairs = pairs.numpy()
    fa_dict = {n: [None, int(ln), 1] for n, ln in zip(asm.names, asm.lengths.tolist())}
    args = Namespace(flank=60 if bin_kb else 500)
    if not bin_kb:
        names = list(fa_dict)
        table, _ = cluster.count_links([pairs], names, asm.lengths, set(names), args.flank, want_clm=False)
        return table, names
    bin_size = bin_kb * 1000
    split = {n for n, v in fa_dict.items() if v[1] > bin_size}
    frag_len = {}
    for n, v in fa_dict.items():
        if n in split:
            nb = ceil(v[1] / bin_size)
            for k in range(nb):
                frag_len["{}_bin{}".format(n, k + 1)] = v[1] - k * bin_size if k + 1 == nb else bin_size
        else:
            frag_len[n] = v[1]
    st = cluster._stream_bins([pairs], fa_dict, args, bin_size, frag_len, set(frag_len), split)
    st["table"].close()
    return st["ftab"], st["frag_names"]


def _haplotypes(names, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(0, 2, len(names)).astype(np.int32)


def _host(table, names, frag_set, hap, w, normalize):
    from haphic_b200 import cluster
    from haphic_b200.links import link_dicts
    _full, flank, _ht, totals = link_dicts(table, names)
    if normalize:
        cluster.normalize_by_nlinks(flank, totals)
    if hap is not None and w:
        cluster.reduce_inter_hap_HiC_links(flank, {n: (int(h), 0) for n, h in zip(names, hap.tolist())}, w)
    m, index = cluster.dict_to_matrix(flank, frag_set, dense_matrix=False, add_self_loops=True)
    m = sp.csc_matrix(m)
    m.sort_indices()
    return m, index, flank


def _device(table, names, frag_set, hap, w, normalize):
    from haphic_b200 import cluster
    mat, index = cluster.device_matrix(table, names, frag_set, normalize_by_nlinks=normalize, add_self_loops=True, hap=hap,
                                       phasing_weight=w)
    m = mat.to_scipy()
    mat.close()
    m.sort_indices()
    return m, index


def _same(a, b):
    assert a.shape == b.shape
    assert np.array_equal(a.indptr, b.indptr)
    assert np.array_equal(a.indices, b.indices)
    assert np.array_equal(a.data.astype(np.float32).view(np.uint32), b.data.astype(np.float32).view(np.uint32))


@pytest.fixture(scope="module")
def ctx():
    from haphic_b200 import cluster
    return cluster._context()


@pytest.mark.parametrize("bins", [False, True])
@pytest.mark.parametrize("normalize", [False, True])
@pytest.mark.parametrize("w", [1.0, 0.5, 0.25])
def test_phased_matrix_matches_host_dict_to_matrix(ctx, bins, normalize, w):
    table, names = _table(ctx, 60 if bins else 160, 300000 if bins else 50000, 120000, 1400 + bins, 120 if bins else 0)
    hap = _haplotypes(names, 7)
    frag_set = {n for k, n in enumerate(names) if k % 7 != 3}
    # a fragment on a haplotype of its own loses every link at w = 1; the ends of the first flank entry are put on two
    # haplotypes, so at w = 1 that entry (which defines the first index) is deleted
    _host0, _i0, flank = _host(table, names, frag_set, None, 0.0, False)
    ids = {n: k for k, n in enumerate(names)}
    first = next(k for k in flank if k[0] in frag_set and k[1] in frag_set)
    hap[ids[first[0]]], hap[ids[first[1]]] = 0, 1
    lonely = next(n for n in names if n in frag_set and n not in first)
    hap[ids[lonely]] = 5
    want, want_index, _ = _host(table, names, frag_set, hap, w, normalize)
    got, got_index = _device(table, names, frag_set, hap, w, normalize)
    assert got_index == want_index
    assert list(got_index.items()) == list(want_index.items())
    _same(got, want)
    if w == 1.0:
        n_linked = sum(1 for n in frag_set if want.getcol(want_index[n]).nnz > 1)
        assert want_index[lonely] >= n_linked                  # in the unlinked tail
        assert want[want_index[first[0]], want_index[first[1]]] == 0
    table.close()


def test_phasing_noops_give_the_unphased_matrix(ctx):
    table, names = _table(ctx, 160, 50000, 120000, 1500, 0)
    frag_set = set(names)
    base, base_index = _device(table, names, frag_set, None, 0.0, False)
    one = np.zeros(len(names), np.int32)                       # one GFA file: every contig on haplotype 0
    for hap, w in ((one, 1.0), (_haplotypes(names, 3), 0.0)):
        got, index = _device(table, names, frag_set, hap, w, False)
        assert list(index.items()) == list(base_index.items())
        _same(got, base)
    table.close()


def test_c2_shape_phased_matrix_against_torch(ctx):
    """10k contigs, 50M pairs, two haplotypes: the device matrix against a torch reconstruction from the fetched table
    (flank mask, keep mask, the same fp64 x - x * w, first-seen indices by the smallest touch)."""
    import torch
    from haphic_b200 import cluster
    table, names = _table(ctx, 10000, 20000, 50_000_000, 1600, 0, device="cuda")
    dev = torch.device("cuda", ctx.device)
    f = table.fetch()
    ki = torch.from_numpy(f["key_i"].astype(np.int64)).to(dev)
    kj = torch.from_numpy(f["key_j"].astype(np.int64)).to(dev)
    flank = torch.from_numpy(f["flank"].astype(np.int64)).to(dev)
    touch_t = torch.from_numpy(f["first_flank"].astype(np.int64)).to(dev) * 2
    n = len(names)
    hap_np = _haplotypes(names, 11)
    hap = torch.from_numpy(hap_np.astype(np.int64)).to(dev)
    keep_np = np.arange(n) % 10 != 4
    keep = torch.from_numpy(keep_np).to(dev)
    frag_set = {nm for nm, k in zip(names, keep_np.tolist()) if k}
    for w in (1.0, 0.5):
        x = flank.to(torch.float64)
        inter = hap[ki] != hap[kj]
        x = torch.where(inter, x - x * w, x)
        sel = (flank > 0) & keep[ki] & keep[kj] & (x != 0)
        big = torch.iinfo(torch.int64).max
        touch = torch.full((n,), big, dtype=torch.int64, device=dev)
        touch.scatter_reduce_(0, ki[sel], touch_t[sel], "amin")
        touch.scatter_reduce_(0, kj[sel], touch_t[sel] + 1, "amin")
        linked = touch < big
        order = torch.argsort(touch[linked], stable=True)
        index = torch.full((n,), -1, dtype=torch.int64, device=dev)
        index[torch.nonzero(linked).squeeze(1)[order]] = torch.arange(int(linked.sum()), device=dev)
        got, got_index = _device(table, names, frag_set, hap_np, w, False)
        idx_np = index.cpu().numpy()
        for c in np.nonzero(idx_np >= 0)[0].tolist():
            assert got_index[names[c]] == idx_np[c]
        full_index = np.array([got_index.get(nm, -1) for nm in names], np.int64)
        fi = torch.from_numpy(full_index).to(dev)
        r, c, v = fi[ki[sel]], fi[kj[sel]], x[sel].to(torch.float32)
        m = len(frag_set)
        rows = torch.cat([r, c, torch.arange(m, device=dev)]).cpu().numpy()
        cols = torch.cat([c, r, torch.arange(m, device=dev)]).cpu().numpy()
        vals = torch.cat([v, v, torch.ones(m, dtype=torch.float32, device=dev)]).cpu().numpy()
        want = sp.csc_matrix((vals, (rows, cols)), shape=(m, m))
        want.sort_indices()
        _same(got, want)
    table.close()


def test_fractional_weight_matrix_takes_the_weights_encoding(ctx):
    from haphic_b200 import cluster
    from haphic_b200.mcl import Mcl
    from tests.test_gpu_gemm import exact_m1
    table, names = _table(ctx, 600, 30000, 400000, 1700, 0)
    hap = _haplotypes(names, 13)
    mat, _index = cluster.device_matrix(table, names, set(names), add_self_loops=True, hap=hap, phasing_weight=0.3)
    host = mat.to_scipy()
    assert np.any(host.data != np.round(host.data))            # fractional values present
    mc = Mcl(mat, preexp="dense")
    assert mc.preexp["mode"] == "dense" and mc.preexp["a_planes"] == 3 and mc.preexp["passes"] == 6
    m1 = mc.m1().astype(np.float64)
    exact = exact_m1(host)
    nz = exact != 0
    assert np.array_equal(m1 != 0, nz)
    assert (np.abs(m1[nz] - exact[nz]) / exact[nz]).max() <= 2e-6
    mc.close()
    mat.close()
    table.close()
