"""CPU checks of `haphic plot`: the host AGP layout against the reference's goldens, the argument defaults, the pickle
format and its checks, and the numpy bnewt oracle against the reference's x and step counts."""

import argparse
import ast
import os
import pickle

import numpy as np
import pytest

from haphic_b200 import plot
from tests import plot_oracle

CASES = ("main", "specified", "allkept", "error")


def golden(golden_dir, tag):
    return np.load(os.path.join(golden_dir, "plot_{}.npz".format(tag)))


def write_case(z, tmp_path):
    agp = tmp_path / "asm.agp"
    agp.write_text(str(z["agp"]))
    return str(agp)


def layout_of(z, agp):
    spec = str(z["specified"]) or None
    return plot.Layout(agp, int(z["bin_size"]) * 1000, int(z["min_len"]), spec)


@pytest.mark.parametrize("tag", CASES)
def test_layout_resolves_every_golden_position(golden_dir, tmp_path, tag):
    z = golden(golden_dir, tag)
    L = layout_of(z, write_case(z, tmp_path))
    assert L.group_list == list(z["group_list"])
    assert L.nb == int(z["nb"])
    assert sorted(n for n, f in zip(L.names, L.in_set) if f) == list(z["in_ctg_set"])
    got = []
    for c, p in zip(z["probe_ctg"], z["probe_pos"]):
        b = L.resolve(str(c), int(p))
        got.append(-1 if b is None else b)
    assert got == z["probe_bin"].tolist()


def test_layout_covers_the_edge_cases(golden_dir):
    z = golden(golden_dir, "main")
    bins = dict(zip(zip(z["probe_ctg"].tolist(), z["probe_pos"].tolist()), z["probe_bin"].tolist()))
    assert bins[("C", 2000010)] == -1            # listed aln bin, no range contains it
    e = golden(golden_dir, "error")
    assert -2 in e["probe_bin"].tolist()         # positions the reference cannot place
    assert "C:1500007" in str(e["error"]) and str(e["error"]).endswith(".pairs files match")


def test_ceil_quirk_blocks(golden_dir, tmp_path):
    z = golden(golden_dir, "allkept")
    L = layout_of(z, write_case(z, tmp_path))
    # S2 ends on an exact multiple of the bin size: its block has one bin fewer than its share of the matrix
    sizes = [L.group_size[g] // L.bin_size + 1 for g in L.group_list]
    blocks = L.blocks()
    assert sum(sizes) == L.nb
    assert any(n != s for (_o, n), s in zip(blocks, sizes))
    assert blocks[1][0] == sizes[0] - (sizes[0] - blocks[0][1])


def test_argument_defaults_match_the_reference_order(golden_dir):
    z = golden(golden_dir, "main")
    ref_items = ast.literal_eval(str(z["pkl_args"]))
    args = plot.parse_arguments([ref_items[0][1], ref_items[1][1], "--bin_size", "100", "--min_len", "1",
                                 "--normalization", "KR"])
    assert list(vars(args)) == [k for k, _ in ref_items]
    defaults = dict(ref_items)
    for k, v in vars(args).items():
        if k not in ("agp", "alignments"):
            assert v == defaults[k], k
    assert len(vars(args)) == 29


def test_pickle_round_trip_and_checks(golden_dir, tmp_path, monkeypatch):
    z = golden(golden_dir, "main")
    agp = write_case(z, tmp_path)
    monkeypatch.chdir(tmp_path)
    args = plot.parse_arguments([agp, "x.pairs", "--bin_size", "100"])
    plot.output_pickle(z["matrix"], args)
    mat, a2, md5 = pickle.load(open("contact_matrix.pkl", "rb"))
    assert np.array_equal(mat, z["matrix"]) and md5 == str(z["pkl_md5"]) and vars(a2) == vars(args)
    assert np.array_equal(plot.load_pickle("contact_matrix.pkl", args), z["matrix"])
    bad = argparse.Namespace(**dict(vars(args), min_len=2))
    with pytest.raises(RuntimeError, match=r"The input parameters \(--bin_size 100 --min_len 2 --specified_scaffolds None\) "
                                           r"are not consistent with those used to generate `contact_map.pkl` "
                                           r"\(--bin_size 100 --min_len 1 --specified_scaffolds None\)"):
        plot.load_pickle("contact_matrix.pkl", bad)
    other = tmp_path / "other.agp"
    other.write_text(str(z["agp"]) + "\n")
    with pytest.raises(RuntimeError, match="The AGP file used to generate contact_matrix.pkl .* is different from the input AGP"):
        plot.load_pickle("contact_matrix.pkl", argparse.Namespace(**dict(vars(args), agp=str(other))))


def test_numpy_bnewt_oracle_matches_the_reference(golden_dir):
    z = np.load(os.path.join(golden_dir, "plot_bnewt.npz"))
    for name in z["names"]:
        x, outer, inner = plot_oracle.bnewt(z["A_" + name])
        assert [outer, inner] == z["steps_" + name].tolist(), name
        np.testing.assert_allclose(x, z["x_" + name], rtol=1e-12, err_msg=name)
