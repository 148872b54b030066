"""CPU checks of assembly correction: the `portion` stand-in the correction goldens were made with, the numpy oracle
against the reference's own results, and the host bookkeeping (piece names, fa_dict order, break tables)."""

import json
import os
import sys

import numpy as np

from tests import correct_oracle as orc
from tests.util import GOLDEN, load_golden

sys.path.insert(0, GOLDEN)
import _portion as P  # noqa: E402


def test_portion_standin_semantics():
    u = P.closed(0, 5) | P.closed(5, 10) | P.closed(20, 30)
    assert len(u) == 2 and u.lower == 0 and u.upper == 30
    assert [(i.lower, i.upper) for i in u] == [(0, 10), (20, 30)]
    assert len(P.closed(0, 5) | P.closed(6, 10)) == 2              # a gap: not merged
    v = P.closed(0, 30) - u
    assert len(v) == 1 and (v.lower, v.upper) == (10, 20)
    assert not v.overlaps(P.closed(20, 25)) and v.overlaps(P.closed(19, 25))
    assert P.closed(3, 4).overlaps(P.closed(4, 9)) and not P.closed(3, 4).overlaps(P.closed(5, 9))
    assert len(P.empty()) == 0 and len(P.empty() | P.closed(1, 2)) == 1
    w = P.closed(0, 100) - (P.closed(0, 10) | P.closed(40, 50) | P.closed(90, 100))
    assert [(i.lower, i.upper) for i in w] == [(10, 40), (50, 90)]


def test_oracle_detect_matches_reference_cases():
    g = load_golden("correct_detect.npz")
    want = json.loads(str(g["breaks_json"]))
    for name, length, cov in zip(g["names"].tolist(), g["lengths"].tolist(), json.loads(str(g["cov_json"]))):
        got = [[p, c] for p, c in orc.detect(np.array(cov, np.int32), length, 500)]
        assert got == want.get(name, []), name


def test_oracle_matches_reference_rounds():
    """Every round's coverage and breakpoints, from the records alone (items 1-3)."""
    from haphic_b200 import synth
    n_zero = n_multi = n_nonzero = 0
    for tag in ("r1", "r2", "r4", "r4g3", "r4g3_nogap"):
        g = load_golden("correct_{}.npz".format(tag))
        nchr, n_contigs, mean_len, n_pairs, n_joins, span, seed, group, gap = json.loads(str(g["case_json"]))
        kw = json.loads(str(g["argkw"]))
        asm, pairs, _j = synth.chimera_case(nchr, n_contigs, mean_len, n_pairs, n_joins, span, seed, group=group, gap=gap)
        want = json.loads(str(g["rounds_json"]))
        got = orc.correct_rounds(pairs, asm.lengths, kw.get("correct_resolution", 500), kw["correct_nrounds"])
        assert len(got) == len(want), tag
        for (covs, brk), w in zip(got, want):
            assert [c.tolist() for c in covs] == w["cov"], tag
            assert [[w["names"][i], [[p, c] for p, c in b]] for i, b in brk] == w["breaks"], tag
            n_zero += sum(1 for _i, b in brk for _p, c in b if c == 0)
            n_multi += sum(1 for _i, b in brk if len(b) > 1)
            n_nonzero += sum(1 for _i, b in brk for _p, c in b if c != 0)
    # the fixtures reach the zero-coverage path with several breakpoints in one fragment, and the non-zero path
    assert n_zero >= 4 and n_multi >= 2 and n_nonzero >= 2, (n_zero, n_multi, n_nonzero)


def test_host_bookkeeping_matches_reference(tmp_path, monkeypatch):
    """break_and_update_ctgs' fa_dict / table updates and the output files from the reference's own breakpoints."""
    from haphic_b200 import cluster, correct, synth
    for tag in ("r1", "r2", "r4g3", "r4g3_nogap"):
        g = load_golden("correct_{}.npz".format(tag))
        nchr, n_contigs, mean_len, n_pairs, n_joins, span, seed, group, gap = json.loads(str(g["case_json"]))
        asm, _pairs, _j = synth.chimera_case(nchr, n_contigs, mean_len, 10, n_joins, span, seed, group=group, gap=gap)
        d = tmp_path / tag
        d.mkdir()
        monkeypatch.chdir(d)
        synth.write_fasta(asm, "asm.fa", seed=seed + 5)
        fa_dict = cluster.parse_fasta("asm.fa")
        unbroken = set(fa_dict)
        src, pos, frag = {}, {}, {}
        rounds = [r for r in json.loads(str(g["rounds_json"])) if r["breaks"]]
        for k, r in enumerate(rounds):
            if k == 0:
                for name, _b in r["breaks"]:
                    src[name], pos[name], frag[name] = name, [0], [name]
            correct.break_and_update_ctgs([(n, [p for p, _c in b]) for n, b in r["breaks"]], src, pos, frag, fa_dict, unbroken,
                                          lambda s: cluster.count_RE_sites(s, "GATC"))
            unbroken -= {n for n, _b in r["breaks"]}
        assert [[k, v[1], v[2]] for k, v in fa_dict.items()] == json.loads(str(g["fa_json"]))
        assert pos == json.loads(str(g["final_pos_json"])) and frag == json.loads(str(g["final_frag_json"]))
        correct.write_corrected_files(fa_dict, unbroken, len(rounds[0]["breaks"]), "asm.fa")
        with open("corrected_ctgs.txt") as f:
            assert f.read() == str(g["corrected_ctgs"])


def test_piece_names_shift_to_source_coordinates():
    from haphic_b200.correct import piece_names
    assert piece_names("c", [100, 250], 400, {"c"}) == ["c:1-100", "c:101-250", "c:251-400"]
    assert piece_names("c:101-400", [150], 300, set()) == ["c:101-250", "c:251-400"]
