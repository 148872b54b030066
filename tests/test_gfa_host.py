"""Host side of `haphic cluster --gfa` against what the unmodified reference computed (tests/golden/gfa_*.npz, made by
tests/golden/make_gfa_golden.py): parse_gfa and its messages, the read-depth filter of filter_fragments,
reduce_inter_hap_HiC_links on the frozen dicts (value types included), the fp64 pass over the full links' arrays with the
full_links.pkl writer, and the --phasing_weight range check.  No GPU."""

import json
import logging
import os
import pickle
import subprocess
import sys
from collections import defaultdict

import numpy as np
import pytest

from tests.util import load_golden

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RUNS = ["w1", "w05_norm", "one_x", "one_frac", "bins", "allelic", "correct"]
PHASED = ["w1", "w05_norm", "bins", "allelic", "correct"]


def value(text):
    """repr of an int or a float back to the same Python object."""
    return float(text) if any(c in text for c in ".eEn") else int(text)


def typed_dict(items):
    d = defaultdict(int)
    for *key, v in items:
        d[tuple(key) if len(key) > 1 else key[0]] = value(v)
    return d


def typed_items(d):
    return [list(k) + [repr(v)] for k, v in d.items()]


def golden_json(g, key):
    """A JSON member of a gfa_*.npz fixture (stored as UTF-8 bytes)."""
    return json.loads(g[key].tobytes().decode())


def record(tag):
    return golden_json(load_golden("gfa_{}.npz".format(tag)), "record_json")


class Capture(logging.Handler):
    def __init__(self):
        super().__init__()
        self.lines = []

    def emit(self, r):
        self.lines.append((r.funcName, r.levelname, r.getMessage()))


@pytest.fixture
def capture():
    from haphic_b200 import cluster
    h = Capture()
    cluster.logger.addHandler(h)
    yield h
    cluster.logger.removeHandler(h)


@pytest.mark.parametrize("tag", ["ok", "bad_len", "missing", "extra"])
def test_parse_gfa_matches_reference(tmp_path, capture, tag):
    from haphic_b200 import cluster
    g = golden_json(load_golden("gfa_parse.npz"), "parse_json")
    case = g[tag]
    paths = []
    for name in case["file_order"]:
        (tmp_path / name).write_text(case["files"][name])
        paths.append(str(tmp_path / name))
    fa = {n: [None, ln, 1] for n, ln in g["fa"].items()}
    if case["error"] is None:
        got = cluster.parse_gfa(paths, fa)
        assert list(got) == case["order"]
        assert {k: list(v) for k, v in got.items()} == case["result"]
    else:
        with pytest.raises(RuntimeError) as e:
            cluster.parse_gfa(paths, fa)
        # the messages name the GFA path: compare them with the directory taken out
        assert str(e.value).replace(str(tmp_path) + os.sep, "") == case["error"].replace(_golden_dir(case["error"]), "")
    got_logs = ["{} {}".format(lv, msg).replace(str(tmp_path) + os.sep, "") for _f, lv, msg in capture.lines]
    want_logs = [ln.replace(_golden_dir(ln), "") for ln in case["logs"]]
    assert got_logs == want_logs
    assert all(f == "parse_gfa" for f, _lv, _m in capture.lines)


def _golden_dir(text):
    """The temporary directory the fixture's GFA paths were in ('' when the text names none)."""
    k = text.find("/tmp")
    if k < 0:
        return ""
    end = text.find(".gfa", k)
    return text[k:text.rfind("/", k, end) + 1]


def test_parse_gfa_keeps_the_sequence_column_whole(tmp_path):
    """A sequence column with tabs-free megabase sequence and extra optional fields after rd:i: parse like hifiasm's."""
    from haphic_b200 import cluster
    seq = "ACGT" * 250000
    (tmp_path / "a.gfa").write_text("S\tc1\t{}\tLN:i:1000000\trd:i:17\tXX:Z:tail\nS\tc2\t*\tLN:i:5\trd:i:3\n".format(seq))
    got = cluster.parse_gfa([str(tmp_path / "a.gfa")], {"c1": [None, 1000000, 1], "c2": [None, 5, 1]})
    assert got == {"c1": (0, 17), "c2": (0, 3)}


FILTER_DRIVER = r"""
import json, logging, sys
sys.path.insert(0, {repo!r})
import numpy as np
from haphic_b200 import cluster
rec = json.loads(open({path!r}).read())
fin = rec["filter_in"]
def value(t):
    return float(t) if any(c in t for c in ".eEn") else int(t)
flank = {{(a, b): value(v) for a, b, v in fin["flank_link_dict"]}}
lines = []
class H(logging.Handler):
    def emit(self, r):
        lines.append("[{{}}] {{}}".format(r.funcName, r.getMessage()))
cluster.logger.addHandler(H())
got = cluster.filter_fragments(set(fin["Nx_frag_set"]), fin["RE_site_dict"], fin["RE_site_cutoff"], fin["frag_link_dict"],
                               fin["density_lower"], fin["density_upper"], fin["topN"], fin["rank_sum_upper"],
                               fin["rank_sum_hard_cutoff"], flank, {{k: tuple(v) for k, v in fin["read_depth_dict"].items()}},
                               fin["read_depth_upper"], set())
print(json.dumps(dict(out=sorted(got), lines=lines)))
"""


@pytest.mark.parametrize("tag", RUNS)
def test_read_depth_filter_matches_reference(tmp_path, tag):
    """filter_fragments on the host with the inputs the reference got: same fragments, same log lines (the Nx set is
    rebuilt in a PYTHONHASHSEED=0 process, as the fixture's was, so set-iteration orders agree)."""
    g = load_golden("gfa_{}.npz".format(tag))
    rec = golden_json(g, "record_json")
    path = tmp_path / "rec.json"
    path.write_text(json.dumps(rec))
    env = dict(os.environ, PYTHONHASHSEED="0")
    r = subprocess.run([sys.executable, "-c", FILTER_DRIVER.format(repo=REPO, path=str(path))], env=env, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    got = json.loads(r.stdout.splitlines()[-1])
    assert got["out"] == rec["filter_out"]
    want = [ln for ln in golden_json(g, "log_lines") if ln.startswith("[filter_fragments]")]
    assert got["lines"] == want
    assert any("[read depth filtering]" in ln for ln in want)


@pytest.mark.parametrize("tag", PHASED)
@pytest.mark.parametrize("target", ["flank_link_dict", "full_link_dict"])
def test_reduce_inter_hap_links_matches_reference(capture, tag, target):
    from haphic_b200 import cluster
    red = record(tag)["reduce_" + target]
    d = typed_dict(red["before"])
    hap = {k: (v, 0) for k, v in red["hap"].items()}
    cluster.reduce_inter_hap_HiC_links(d, hap, red["weight"], target=target)
    assert typed_items(d) == red["after"]                 # order, values and int / float types
    assert [(f, m) for f, _lv, m in capture.lines] == [
        ("reduce_inter_hap_HiC_links", "Reducing inter-haplotype Hi-C links in {}...".format(target))]


@pytest.mark.parametrize("tag", PHASED)
def test_oracle_reduction_of_arrays_and_pickle_match_reference(tmp_path, tag):
    """The fp64 reduction of the full links on arrays (tests/stats_oracle.py, the host reference of the device's
    hh_links_fetch_phased) gives the reference's dict, and the native writer's full_links.pkl loads as that dict: same
    order, same values, floats and ints where the reference has them."""
    from haphic_b200 import cluster
    from tests.stats_oracle import reduce_phasing
    import __graft_entry__
    __graft_entry__.build()
    g = load_golden("gfa_{}.npz".format(tag))
    red = golden_json(g, "record_json")["reduce_full_link_dict"]
    before = typed_dict(red["before"])
    if any(isinstance(v, float) for v in before.values()):
        pytest.skip("full links already scaled on the host (the dict path)")
    names = sorted({n for k in before for n in k})
    ids = {n: i for i, n in enumerate(names)}
    arr = cluster.LinkArrays(names, [ids[a] for a, _ in before], [ids[b] for _, b in before], list(before.values()))
    hap = np.array([red["hap"][n] for n in names], np.int32)
    arr = reduce_phasing(arr, hap, red["weight"])
    assert typed_items(arr.to_dict()) == red["after"]
    want = golden_json(g, "full_links_items")
    assert typed_items(arr.to_dict()) == want
    arr.write_pickle(str(tmp_path / "full_links.pkl"))
    with open(tmp_path / "full_links.pkl", "rb") as f:
        loaded = pickle.load(f)
    assert type(loaded) is defaultdict and loaded.default_factory is int
    assert typed_items(loaded) == want


def test_phasing_weight_outside_unit_interval_is_rejected(tmp_path):
    from haphic_b200 import cluster
    args = cluster.parse_arguments([str(tmp_path / "asm.fa"), str(tmp_path / "aln.pairs"), "2", "--gfa", "a.gfa,b.gfa",
                                    "--phasing_weight", "1.5"])
    with pytest.raises(ValueError, match="phasing_weight"):
        cluster.run(args)
    args.phasing_weight = -0.25
    with pytest.raises(ValueError, match="phasing_weight"):
        cluster.run(args)
