"""`haphic cluster --gfa` with a fractional --phasing_weight on the device: the contig-level full-link reduction
(hh_links_fetch_phased) and the reassignment statistics over int / float links (hh_stats):
  * whole runs on the reference's fixtures write the same statistics files and full_links.pkl items with the host versions
    of both steps disabled, so the device path is what produced them;
  * device against host (LinkArrays.reduce_phasing, _ranked_group_links_mixed / _best_group_statistics with
    HAPHIC_STATS_DEVICE=0), fp64 bit for bit, on a 10k-contig two-haplotype input and on hand-made edge cases;
  * one inflation's statistics at the C3 shape (50k contigs, 200M pairs, w = 0.5) equal the host path's."""

import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

from tests.test_gfa_host import golden_json
from tests.util import load_golden

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

DRIVER = r"""
import sys
sys.path.insert(0, {repo!r})
from haphic_b200 import cluster, synth

def host_step(*a, **k):
    raise AssertionError("host step ran on the device path")

cluster.LinkArrays.reduce_phasing = host_step
cluster._ranked_group_links_mixed = host_step
gfa = synth.gfa_case(*{case!r}, ".", bam={bam!r})
argv = ["asm.fa", "aln.bam" if {bam!r} else "aln.pairs", str({nchr})] + {extra!r} + ["--gfa", ",".join(gfa)]
cluster.run(cluster.parse_arguments(argv), log_file="HapHiC_cluster.log")
"""


def typed_items(d):
    return [list(k) + [repr(v)] for k, v in d.items()]


@pytest.mark.parametrize("tag,bam", [("w05_norm", False), ("w05_norm", True), ("w1", False), ("bins", False)])
def test_run_on_the_device_path_matches_reference(tmp_path, tag, bam):
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
    want = {p: t for p, t in golden_json(g, "files_json").items() if p.startswith("inflation_")}
    stats = [p for p in want if p.endswith("_statistics.txt")]
    assert stats
    for p in sorted(want):
        assert (tmp_path / p).read_text() == want[p], p
    with open(tmp_path / "full_links.pkl", "rb") as f:
        assert typed_items(pickle.load(f)) == golden_json(g, "full_links_items")


# ------------------------------------------------------------------------------------------------
# device against host
# ------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def ctx():
    from haphic_b200 import cluster
    return cluster._context()


def _bits(x):
    return np.ascontiguousarray(x, dtype=np.float64).view(np.uint64)


def _table(names, lengths, pairs):
    from haphic_b200 import cluster
    table, _ = cluster.count_links([pairs], names, lengths, set(names), 500, want_clm=False)
    return table


def _host_arrays(table, names, hap, w):
    from haphic_b200 import cluster
    f = table.fetch()
    arr = cluster.LinkArrays(names, f["key_i"], f["key_j"], f["full"])
    arr.reduce_phasing(hap, w)
    return arr


def _same_arrays(dev, host):
    assert np.array_equal(dev.key_i, host.key_i) and np.array_equal(dev.key_j, host.key_j)
    assert (dev.is_float is None) == (host.is_float is None)
    if host.is_float is None:
        assert dev.values.dtype == np.int64 and np.array_equal(dev.values, host.values)
    else:
        assert np.array_equal(dev.is_float, host.is_float)
        assert np.array_equal(_bits(dev.values), _bits(host.values))


def _typed(lst):
    return [(c, type(v).__name__, repr(v)) for c, v in lst]


def _compare_statistics(monkeypatch, fa_dict, links, ctg_group, group_RE):
    """Ranking and the three statistic lists on the device against the host path (HAPHIC_STATS_DEVICE=0)."""
    from haphic_b200 import cluster
    monkeypatch.setenv("HAPHIC_STATS_DEVICE", "1")
    dev_rank = cluster._ranked_group_arrays(links, ctg_group)
    dev_best = cluster._best_group_statistics(fa_dict, links, ctg_group, group_RE)
    monkeypatch.setenv("HAPHIC_STATS_DEVICE", "0")
    host_rank = cluster._ranked_group_arrays(links, ctg_group)
    host_best = cluster._best_group_statistics(fa_dict, links, ctg_group, group_RE)
    monkeypatch.setenv("HAPHIC_STATS_DEVICE", "1")
    if host_rank is None:
        assert dev_rank is None
    else:
        _gid, hc, hg, hs, hf = host_rank
        _gid, dc, dg, ds, df = dev_rank
        assert np.array_equal(dc, hc) and np.array_equal(dg, hg)
        assert np.array_equal(_bits(ds), _bits(hs))
        assert (df is None) == (hf is None)
        if hf is not None:
            assert np.array_equal(np.asarray(df, bool), np.asarray(hf, bool))
    for d, h in zip(dev_best, host_best):
        assert _typed(d) == _typed(h)
    return dev_best


@pytest.fixture(scope="module")
def synthetic(ctx):
    """10k contigs on 24 chromosomes, two haplotypes (odd / even chromosome), 4M pairs with allelic links."""
    import torch
    from haphic_b200 import synth
    asm = synth.make_assembly(24, 10000, 20000, seed=77)
    pairs = synth.make_pairs(asm, 4_000_000, seed=78, homolog=(2, 0.2), device=torch.device("cuda", ctx.device))
    names = list(asm.names)
    table = _table(names, asm.lengths, pairs.cpu().numpy())
    hap = (asm.chrom % 2).astype(np.int32)
    rng = np.random.default_rng(79)
    group = np.where(rng.random(asm.n) < 0.9, asm.chrom // 2 + 12 * (rng.random(asm.n) < 0.05), -1)
    ng = int(group.max()) + 1
    ctg_group = {nm: ("ungrouped" if g < 0 else int(g)) for nm, g in zip(names, group.tolist())}
    group_RE = {g: int(rng.integers(2, 4000)) for g in range(ng)}
    fa_dict = {nm: [None, int(ln), int(rng.integers(1, 300))] for nm, ln in zip(names, asm.lengths.tolist())}
    yield dict(table=table, names=names, hap=hap, ctg_group=ctg_group, group_RE=group_RE, fa_dict=fa_dict)
    table.close()


@pytest.mark.parametrize("w", [0.5, 0.25, 0.1, 1.0])
def test_synthetic_reduction_and_statistics_match_host(monkeypatch, synthetic, w):
    from haphic_b200 import cluster
    s = synthetic
    dev = cluster.LinkArrays.from_phased(s["names"], s["table"].fetch_phased(s["hap"], w))
    host = _host_arrays(s["table"], s["names"], s["hap"], w)
    _same_arrays(dev, host)
    if w == 1.0:
        assert dev.is_float is None and len(dev) < int(s["table"].info.nnz_full)        # the inter-haplotype links are gone
    else:
        assert dev.is_float.any() and not dev.is_float.all()
    _compare_statistics(monkeypatch, s["fa_dict"], dev, s["ctg_group"], s["group_RE"])


def test_two_rounding_form_is_what_runs(ctx):
    """9 links between haplotypes at w = 0.3: 9 - 9 * 0.3 = 6.300000000000001, while 9 * (1 - 0.3) and a fused
    multiply-add both give 6.3."""
    from fractions import Fraction
    from haphic_b200 import cluster
    names = ["a", "b", "c"]
    rec = np.array([[0, 10, 1, 20]] * 9 + [[0, 30, 2, 40]] * 5, np.int32)
    table = _table(names, np.array([1000, 1000, 1000], np.int64), rec)
    got = cluster.LinkArrays.from_phased(names, table.fetch_phased(np.array([0, 1, 0], np.int32), 0.3))
    table.close()
    assert got.python_values() == [9 - 9 * 0.3, 5]
    assert [type(v) for v in got.python_values()] == [float, int]
    assert got.values[0] != 9 * (1 - 0.3)
    assert got.values[0] != float(Fraction(9) - Fraction(9) * Fraction(0.3))     # fused: one rounding


def _links(n, entries, floats):
    """LinkArrays over contigs c0..c{n-1} from (i, j, value) triples; ``floats`` = is_float per entry (None: all ints)."""
    from haphic_b200 import cluster
    names = ["c{}".format(k) for k in range(n)]
    ki, kj, v = zip(*entries)
    return names, cluster.LinkArrays(names, ki, kj, np.array(v, np.float64 if floats is not None else np.int64),
                                     None if floats is None else np.array(floats, bool))


def test_edge_cases_match_host(monkeypatch, ctx):
    from haphic_b200 import cluster
    rng = np.random.default_rng(5)
    # contigs 0..9: groups 0 / 1 / 2 (c0..c2 in group 0, c3..c5 in 1, c6, c7 in 2), c8 / c9 ungrouped.
    # c0: tie between groups 1 and 2 (2.5 each), group 2 met first; c8: links only to ungrouped c9.
    ent = [(0, 6, 1.25), (0, 3, 2.5), (0, 7, 1.25), (1, 4, 3), (1, 2, 0.1), (1, 5, 0.2), (8, 9, 7), (5, 9, 0.7),
           (2, 6, 0.30000000000000004), (4, 7, 11)]
    groups = {0: 0, 1: 0, 2: 0, 3: 1, 4: 1, 5: 1, 6: 2, 7: 2}
    for floats in ([True, True, True, False, True, True, False, True, True, False],      # mixed
                   [True] * len(ent),                                                    # every link a float
                   [False] * len(ent)):                                                  # no float at all
        vals = [v if f else max(1, int(v)) for (_i, _j, v), f in zip(ent, floats)]
        names, links = _links(10, [(i, j, v) for (i, j, _), v in zip(ent, vals)], floats)
        ctg_group = {nm: groups.get(k, "ungrouped") for k, nm in enumerate(names)}
        fa_dict = {nm: [None, 1000 + k, 3 + k] for k, nm in enumerate(names)}
        best = _compare_statistics(monkeypatch, fa_dict, links, ctg_group, {0: 7, 1: 9, 2: 13})
        assert best[0][8] == ("c8", 0)                                                   # linked only to ungrouped
        ranked = cluster.ranked_group_links(links, ctg_group)
        assert [g for g, _ in ranked["c0"]][:2] == [2, 1]                                 # the tie: first visit wins
    # one group only: others = 0, ratio 1000000
    names, links = _links(4, [(0, 1, 2.5), (0, 2, 1.5), (1, 3, 4.0)], [True, True, False])
    ctg_group = {"c0": 0, "c1": 0, "c2": 0, "c3": 0}
    fa_dict = {nm: [None, 1000, 5] for nm in names}
    best = _compare_statistics(monkeypatch, fa_dict, links, ctg_group, {0: 20})
    assert all(v == 1000000 for _c, v in best[2])
    # long segments: c0 has 1500 float links into group 0 (> 1024 terms in one sum) and 40 into group 1 (> 32); c1 is linked to
    # 1200 groups (a ranked list of > 1024 groups for the compensated sum)
    ent, flt = [], []
    n = 3000
    for k in range(1500):
        ent.append((0, 2 + k, float(rng.random() * 10.0 ** rng.integers(-3, 4))))
        flt.append(True)
    for k in range(40):
        ent.append((0, 1502 + k, int(rng.integers(1, 9))))
        flt.append(False)
    for k in range(1200):
        ent.append((1, 1600 + k, float(rng.random() * 10.0 ** rng.integers(-2, 3))))
        flt.append(bool(k % 3))
    vals = [v if f else int(v) for (_i, _j, v), f in zip(ent, flt)]
    names, links = _links(n, [(i, j, v) for (i, j, _), v in zip(ent, vals)], flt)
    group = {}
    for k in range(2, 1502):
        group[k] = 0
    for k in range(1502, 1542):
        group[k] = 1
    for k in range(1200):
        group[1600 + k] = 2 + k
    ctg_group = {nm: group.get(k, "ungrouped") for k, nm in enumerate(names)}
    ctg_group["c0"], ctg_group["c1"] = 0, 5
    group_RE = {g: 3 + (g * 7919) % 5000 for g in range(1202)}
    fa_dict = {nm: [None, 1000, 2 + k % 50] for k, nm in enumerate(names)}
    _compare_statistics(monkeypatch, fa_dict, links, ctg_group, group_RE)


def test_c3_shape_statistics_match_host(monkeypatch, ctx):
    """50k contigs, 200M pairs, two haplotypes, w = 0.5 (the shape of scripts/gfa_probe.py): one inflation's device
    statistics against the host path, bit for bit."""
    import torch
    from haphic_b200 import cluster, synth
    from haphic_b200.links import LinkTable, name_rank
    dev = torch.device("cuda", ctx.device)
    asm = synth.make_assembly(24, 50000, 20000, seed=2024)
    names = list(asm.names)
    table = LinkTable(ctx, asm.lengths, name_rank(names), np.ones(asm.n, np.uint8), 500 * 1000)
    step = 1 << 25
    total = 200_000_000
    for lo in range(0, total, step):
        table.add(synth.make_pairs_range(asm, lo, min(total, lo + step), seed=2025, device=dev), stream_offset=lo)
    table.finish()
    hap = (asm.chrom % 2).astype(np.int32)
    links = cluster.LinkArrays.from_phased(names, table.fetch_phased(hap, 0.5))
    table.close()
    assert links.is_float is not None
    per = asm.n // 24
    ctg_group = {nm: k // per for k, nm in enumerate(names)}
    group_RE = {g: 1 + 9 * per for g in range(24)}
    fa_dict = {nm: [None, int(ln), 10] for nm, ln in zip(names, asm.lengths.tolist())}
    monkeypatch.setenv("HAPHIC_STATS_DEVICE", "1")
    dev_best = cluster._best_group_statistics(fa_dict, links, ctg_group, group_RE)
    monkeypatch.setenv("HAPHIC_STATS_DEVICE", "0")
    host_best = cluster._best_group_statistics(fa_dict, links, ctg_group, group_RE)
    for d, h in zip(dev_best, host_best):
        assert _typed(d) == _typed(h)
