"""The reassignment statistics of `haphic cluster` (output_statistics) on the device (hh_stats) for every form of the full
links, and the contig-level full-link reduction of `--gfa` (hh_links_fetch_phased):
  * whole runs on the reference's --gfa fixtures write the same statistics files and full_links.pkl items, and every
    inflation's statistics came from the device;
  * device against the host oracle (tests/stats_oracle.py), fp64 bit for bit, on a 10k-contig two-haplotype input without
    phasing and for w in {0.5, 0.25, 0.1, 1}, and on hand-made edge cases;
  * output_statistics on the same links as the reference's dict (int values, and floats after a
    --remove_concentrated_links-style scaling) and as LinkArrays writes the files of the reference's dict walk;
  * one inflation's statistics at the C3 shape (50k contigs, 200M pairs) on the integer links and after w = 0.5."""

import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

from tests import stats_oracle as so
from tests.test_gfa_host import golden_json
from tests.util import load_golden

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

DRIVER = r"""
import glob, sys
sys.path.insert(0, {repo!r})
from haphic_b200 import cluster, links, synth

calls = []
best = links.GroupLinkStats.best

def counted_best(self, *a, **k):
    calls.append(1)
    return best(self, *a, **k)

links.GroupLinkStats.best = counted_best
gfa = synth.gfa_case(*{case!r}, ".", bam={bam!r})
argv = ["asm.fa", "aln.bam" if {bam!r} else "aln.pairs", str({nchr})] + {extra!r} + ["--gfa", ",".join(gfa)]
cluster.run(cluster.parse_arguments(argv), log_file="HapHiC_cluster.log")
n = len(glob.glob("inflation_*"))
assert n and len(calls) == n, ("inflations", n, "device statistics calls", len(calls))
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
    return so.reduce_phasing(cluster.LinkArrays(names, f["key_i"], f["key_j"], f["full"]), hap, w)


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


def _compare_statistics(ctx, fa_dict, links, ctg_group, group_RE):
    """Ranking and the three statistic lists on the device against the host oracle.  Returns the device's lists and its
    ranking (contig, group)."""
    from haphic_b200 import cluster
    gid, ng = so.group_ids(links.names, ctg_group)
    hc, hg, hs, hf = so.ranked_group_links(links, gid, ng)
    want = so.best_group_statistics(fa_dict, links, ctg_group, group_RE)
    got = cluster._best_group_statistics(fa_dict, links, ctg_group, group_RE)
    dc, dg, ds, df = links.stats_device(ctx).fetch_ranked()          # the ranking the statistics were made from
    assert np.array_equal(dc, hc) and np.array_equal(dg, hg)
    assert np.array_equal(_bits(ds), _bits(hs))                         # integer sums are exact in fp64
    assert np.array_equal(df, np.zeros(len(hc), bool) if hf is None else hf)
    for d, h in zip(got, want):
        assert _typed(d) == _typed(h)
    return got, (dc, dg)


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


@pytest.mark.parametrize("w", [0.5, 0.25, 0.1, 1.0, None])
def test_synthetic_reduction_and_statistics_match_oracle(ctx, synthetic, w):
    """w = None: no phasing, the integer counts of the table."""
    from haphic_b200 import cluster
    s = synthetic
    if w is None:
        f = s["table"].fetch()
        links = cluster.LinkArrays(s["names"], f["key_i"], f["key_j"], f["full"])
    else:
        links = cluster.LinkArrays.from_phased(s["names"], s["table"].fetch_phased(s["hap"], w))
        _same_arrays(links, _host_arrays(s["table"], s["names"], s["hap"], w))
    if w is None or w == 1.0:
        assert links.is_float is None
    if w == 1.0:
        assert len(links) < int(s["table"].info.nnz_full)                    # the inter-haplotype links are gone
    elif w is not None:
        assert links.is_float.any() and not links.is_float.all()
    _compare_statistics(ctx, s["fa_dict"], links, s["ctg_group"], s["group_RE"])


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


def test_edge_cases_match_oracle(ctx):
    rng = np.random.default_rng(5)
    # contigs 0..9: groups 0 / 1 / 2 (c0..c2 in group 0, c3..c5 in 1, c6, c7 in 2), c8 / c9 ungrouped.
    # c0: tie between groups 1 and 2 (2.5 each), group 2 met first; c8: links only to ungrouped c9.
    ent = [(0, 6, 1.25), (0, 3, 2.5), (0, 7, 1.25), (1, 4, 3), (1, 2, 0.1), (1, 5, 0.2), (8, 9, 7), (5, 9, 0.7),
           (2, 6, 0.30000000000000004), (4, 7, 11)]
    groups = {0: 0, 1: 0, 2: 0, 3: 1, 4: 1, 5: 1, 6: 2, 7: 2}
    for floats in ([True, True, True, False, True, True, False, True, True, False],      # mixed
                   [True] * len(ent),                                                    # every link a float
                   [False] * len(ent),                                                   # no float at all
                   None):                                                                # integer links
        vals = [v if f else max(1, int(v)) for (_i, _j, v), f in zip(ent, floats or [False] * len(ent))]
        names, links = _links(10, [(i, j, v) for (i, j, _), v in zip(ent, vals)], floats)
        ctg_group = {nm: groups.get(k, "ungrouped") for k, nm in enumerate(names)}
        fa_dict = {nm: [None, 1000 + k, 3 + k] for k, nm in enumerate(names)}
        best, (rc, rg) = _compare_statistics(ctx, fa_dict, links, ctg_group, {0: 7, 1: 9, 2: 13})
        assert best[0][8] == ("c8", 0)                                                   # linked only to ungrouped
        assert rg[rc == 0][:2].tolist() == [2, 1]                                         # the tie: first visit wins
    # one group only: others = 0, ratio 1000000
    names, links = _links(4, [(0, 1, 2.5), (0, 2, 1.5), (1, 3, 4.0)], [True, True, False])
    ctg_group = {"c0": 0, "c1": 0, "c2": 0, "c3": 0}
    fa_dict = {nm: [None, 1000, 5] for nm in names}
    best, _ = _compare_statistics(ctx, fa_dict, links, ctg_group, {0: 20})
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
    _compare_statistics(ctx, fa_dict, links, ctg_group, group_RE)


def _statistics_files(path, fa_dict, links, clusters):
    from haphic_b200 import cluster
    os.makedirs(path / "inflation_1.5")
    cwd = os.getcwd()
    os.chdir(path)
    try:
        cluster.output_statistics(fa_dict, links, [("1.5", clusters)])
    finally:
        os.chdir(cwd)
    return {fn: (path / "inflation_1.5" / fn).read_text() for fn in sorted(os.listdir(path / "inflation_1.5")) if fn.endswith(".txt")}


def test_statistics_of_dicts_and_arrays_are_the_dict_walk(tmp_path, monkeypatch, ctx):
    """output_statistics on the same links as the reference's dict with int values, as that dict after a
    --remove_concentrated_links-style scaling (floats, integral ones and 0.0 among them) and as LinkArrays: the files are
    the ones the literal dict walk's lists give (ties between groups included), and the dicts are left as they were."""
    from haphic_b200 import cluster
    g = load_golden("links_b.npz")
    names = g["names"].tolist()
    rng = np.random.default_rng(4)
    vals = g["full_vals"].copy()
    vals[rng.random(len(vals)) < 0.5] = 1                       # plenty of ties between groups
    la = cluster.LinkArrays(names, g["full_keys"][:, 0], g["full_keys"][:, 1], vals)
    full = la.to_dict()
    ratio = rng.choice([1.0, 0.0, 0.5, 0.37], len(full)).tolist()
    scaled = {k: v * r for (k, v), r in zip(full.items(), ratio)}
    before = {tag: [(k, repr(v)) for k, v in d.items()] for tag, d in (("full", full), ("scaled", scaled))}
    fa_dict = {n: [None, int(l), int(r)] for n, l, r in zip(names, g["lengths"].tolist(), g["RE_sites"].tolist())}
    lab = rng.integers(-1, 5, size=len(names))
    clusters = [[[n for n, l in zip(names, lab.tolist()) if l == k], 0] for k in range(5)]
    want = {}
    for tag, d in (("full", full), ("scaled", scaled)):
        # the same writer over the literal dict walk's lists
        with monkeypatch.context() as mp:
            mp.setattr(cluster, "_best_group_statistics", lambda fa, _links, cg, gre, d=d: so.statistics_from_dict(fa, d, cg, gre))
            want[tag] = _statistics_files(tmp_path / ("oracle_" + tag), fa_dict, d, clusters)
    assert len(want["full"]) >= 4 and want["full"] != want["scaled"]
    assert _statistics_files(tmp_path / "dict_int", fa_dict, full, clusters) == want["full"]
    assert _statistics_files(tmp_path / "arrays", fa_dict, la, clusters) == want["full"]
    assert _statistics_files(tmp_path / "dict_float", fa_dict, scaled, clusters) == want["scaled"]
    for tag, d in (("full", full), ("scaled", scaled)):
        assert [(k, repr(v)) for k, v in d.items()] == before[tag]


@pytest.fixture(scope="module")
def c3(ctx):
    """The C3 shape of scripts/gfa_probe.py: 50k contigs, 200M pairs, two haplotypes, 24 groups of consecutive contigs."""
    import torch
    from haphic_b200 import synth
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
    per = asm.n // 24
    yield dict(table=table, names=names, hap=(asm.chrom % 2).astype(np.int32),
               ctg_group={nm: k // per for k, nm in enumerate(names)}, group_RE={g: 1 + 9 * per for g in range(24)},
               fa_dict={nm: [None, int(ln), 10] for nm, ln in zip(names, asm.lengths.tolist())})
    table.close()


def test_c3_shape_statistics_match_host(ctx, c3):
    """One inflation's device statistics on the int / float links after w = 0.5 against the host oracle, bit for bit."""
    from haphic_b200 import cluster
    links = cluster.LinkArrays.from_phased(c3["names"], c3["table"].fetch_phased(c3["hap"], 0.5))
    assert links.is_float is not None
    _compare_statistics(ctx, c3["fa_dict"], links, c3["ctg_group"], c3["group_RE"])


def test_c3_shape_integer_statistics_match_host(ctx, c3):
    """The same on the integer links of the unphased run."""
    from haphic_b200 import cluster
    f = c3["table"].fetch()
    links = cluster.LinkArrays(c3["names"], f["key_i"], f["key_j"], f["full"])
    _compare_statistics(ctx, c3["fa_dict"], links, c3["ctg_group"], c3["group_RE"])
