"""Assembly correction (`--correct_nrounds`) on the GPU against the reference's own results (tests/golden/correct_*.npz,
made by tests/golden/make_correction_golden.py) and, at C2 size, against independent torch / numpy restatements."""

import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np
import pytest

from tests import correct_oracle as orc
from tests.util import load_golden

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _args(**kw):
    from haphic_b200 import cluster
    a = cluster.parse_arguments(["asm.fa", "aln.pairs", "4"])
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def test_detect_cases_on_device():
    """The hand-made coverage arrays of correct_detect.npz (median 0, fewer than two high or large runs, small runs inside
    valleys, argmin ties, several zero valleys, the trailing bin), built on the device from single-bin records
    (lo = hi = bin * res, cov[bin] times): the device breakpoints equal the reference's."""
    from haphic_b200 import cluster, correct
    g = load_golden("correct_detect.npz")
    res = 500
    names, lengths = g["names"].tolist(), g["lengths"].astype(np.int64)
    covs = json.loads(str(g["cov_json"]))
    recs = []
    for c, cov in enumerate(covs):
        assert int(lengths[c]) // res + 1 == len(cov)
        for b, k in enumerate(cov):
            recs += [(c, b * res, c, b * res)] * k
    corr = correct.Correction(cluster._context(), lengths, res)
    corr.add(np.array(recs, np.int32))
    assert [v.tolist() for v in corr.coverage().values()] == covs
    corr.round(0.2, 0.1, 5000, True)
    frag, bins, bcov = corr.breaks()
    got = {}
    for f, b, cv in zip(frag.tolist(), bins.tolist(), bcov.tolist()):
        got.setdefault(names[f], []).append([b * res, cv])
    assert got == json.loads(str(g["breaks_json"]))
    corr.close()


@pytest.mark.parametrize("tag", ["r1", "r2", "r4", "r4g3", "r4g3_nogap"])
def test_rounds_match_reference(tmp_path, monkeypatch, tag):
    """Coverage of every examined fragment in every round, breakpoints, fa_dict (names, lengths, RE counts, order), the
    break tables and both output files equal the reference's; the remapped stream equals convert_ctg."""
    from haphic_b200 import cluster, correct, synth
    g = load_golden("correct_{}.npz".format(tag))
    nchr, n_contigs, mean_len, n_pairs, n_joins, span, seed, group, gap = json.loads(str(g["case_json"]))
    asm, pairs, _j = synth.chimera_case(nchr, n_contigs, mean_len, n_pairs, n_joins, span, seed, group=group, gap=gap)
    monkeypatch.chdir(tmp_path)
    synth.write_fasta(asm, "asm.fa", seed=seed + 5)
    args = _args(fasta="asm.fa", **json.loads(str(g["argkw"])))
    fa_dict = cluster.parse_fasta("asm.fa", RE=args.RE)
    src = list(fa_dict.keys())
    corr = correct.Correction(cluster._context(), [fa_dict[n][1] for n in src], args.correct_resolution)
    seen_cov, seen_breaks = [], []
    real_round, real_breaks = corr.round, corr.breaks

    def round_(*a):
        seen_cov.append(list(corr.coverage().values()))
        return real_round(*a)

    def breaks_():
        out = real_breaks()
        seen_breaks.append(out)
        return out

    corr.round, corr.breaks = round_, breaks_
    for k in range(0, len(pairs), 50000):
        corr.add(pairs[k:k + 50000])
    nbroken, final_pos, final_frag = correct.correct_assembly(corr, fa_dict, args, lambda s: cluster.count_RE_sites(s, args.RE))
    rounds = json.loads(str(g["rounds_json"]))
    assert len(seen_cov) == len(rounds)
    res = args.correct_resolution
    for r, want in enumerate(rounds):
        assert len(seen_cov[r]) == len(want["cov"]), r
        for got, exp in zip(seen_cov[r], want["cov"]):
            assert got.tolist() == exp, r
        flat = [(p, c) for _name, lst in want["breaks"] for p, c in lst]
        if flat:
            _f, b, c = seen_breaks[r]
            assert [[int(x) * res, int(y)] for x, y in zip(b, c)] == [list(t) for t in flat], r
    assert nbroken == int(g["nbroken"])
    assert [[k, v[1], v[2]] for k, v in fa_dict.items()] == json.loads(str(g["fa_json"]))
    assert final_pos == json.loads(str(g["final_pos_json"]))
    assert final_frag == json.loads(str(g["final_frag_json"]))
    with open("corrected_ctgs.txt") as f:
        assert f.read() == str(g["corrected_ctgs"])
    with open("corrected_asm.fa") as f:
        assert hashlib.sha1(f.read().encode()).hexdigest() == str(g["corrected_asm_sha1"])
    layout = correct.remap_layout(src, fa_dict, final_pos, final_frag)
    corr.set_layout(*layout)
    assert np.array_equal(corr.remap(pairs), orc.convert(pairs, len(src), layout))
    corr.close()


DRIVER = r"""
import sys
sys.path.insert(0, {repo!r})
from haphic_b200 import cluster, synth, hicio
asm, pairs, _j = synth.chimera_case(*{case!r})
synth.write_fasta(asm, "asm.fa", seed={seed} + 5)
if {bam!r}:
    hicio.write_bam("aln.bam", asm.names, asm.lengths.tolist(), pairs)
    aln = "aln.bam"
else:
    synth.write_pairs(asm, pairs, "aln.pairs")
    aln = "aln.pairs"
args = cluster.parse_arguments(["asm.fa", aln, str({nchr})] + {extra!r})
cluster.run(args, log_file="HapHiC_cluster.log")
"""


@pytest.mark.parametrize("tag,bam", [("run_nobins", False), ("run_nobins", True), ("run_bins", False), ("run_bins", True),
                                     ("run_nobreak", False)])
def test_cluster_run_with_correction_matches_reference(tmp_path, tag, bam):
    import pickle
    g = load_golden("correct_{}.npz".format(tag))
    case = json.loads(str(g["case_json"]))
    extra = []
    for k, v in json.loads(str(g["argkw"])).items():
        extra += ["--" + k, str(v)]
    code = DRIVER.format(repo=REPO, case=tuple(case), seed=case[6], bam=bam, nchr=case[0], extra=extra)
    env = dict(os.environ, PYTHONHASHSEED="0")
    r = subprocess.run([sys.executable, "-c", code], cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    want = json.loads(str(g["files_json"]))
    got = {}
    for root, _d, files in os.walk(tmp_path):
        for fn in files:
            p = os.path.relpath(os.path.join(root, fn), tmp_path)
            if p.endswith(".txt") and (p.startswith("inflation_") or p == "corrected_ctgs.txt"):
                with open(os.path.join(root, fn)) as f:
                    got[p] = f.read()
    assert sorted(got) == sorted(want)
    for p in sorted(want):
        assert got[p] == want[p], p
    assert os.path.islink(tmp_path / "corrected_asm.fa") == bool(g["asm_is_link"])
    with open(tmp_path / "corrected_asm.fa") as f:
        assert hashlib.sha1(f.read().encode()).hexdigest() == str(g["corrected_asm_sha1"])
    with open(tmp_path / "HapHiC_cluster.log") as f:
        log = f.read()
    assert [ln.split("] ", 1)[1] for ln in log.splitlines() if "[recommend_inflation]" in ln] == g["recommend_lines"].tolist()
    assert [ln.split("] ", 1)[1] for ln in log.splitlines() if "[mcl]" in ln] == g["mcl_lines"].tolist()
    with open(tmp_path / "full_links.pkl", "rb") as f:
        full = pickle.load(f)
    assert hashlib.sha1(json.dumps([[a, b, int(v)] for (a, b), v in full.items()]).encode()).hexdigest() == str(g["full_links_sha1"])
    with open(tmp_path / "HT_links.pkl", "rb") as f:
        ht = pickle.load(f)
    assert hashlib.sha1(json.dumps(sorted([a, b, int(v)] for (a, b), v in ht.items())).encode()).hexdigest() == str(g["HT_links_sha1"])
    with open(tmp_path / "paired_links.clm") as f:
        assert hashlib.sha1(f.read().encode()).hexdigest() == str(g["clm_sha1"])
    if not bam:
        with open(tmp_path / "alignments.bed") as f:
            assert hashlib.sha1(f.read().encode()).hexdigest() == str(g["bed_sha1"])


def test_c2_shape_against_torch_and_oracle():
    """10k contigs, 50M pairs, 120 planted chimeras (half with spanning records): coverage = a torch scatter/cumsum,
    breakpoints = the oracle's detection on the fetched coverage, remap = a torch.searchsorted remap."""
    import torch
    from haphic_b200 import cluster, correct, synth
    res = 500
    asm, pairs, junctions = synth.chimera_case(12, 10000, 30000, 50_000_000, 120, 40, 77, device="cuda")
    n = asm.n
    corr = correct.Correction(cluster._context(), asm.lengths, res)
    t0 = time.time()
    for k in range(0, len(pairs), 1 << 24):
        corr.add(pairs[k:k + (1 << 24)])
    cov = corr.coverage()
    print("coverage pass of {} records: {:.2f} s (host copies included)".format(len(pairs), time.time() - t0))
    # independent coverage: torch, global difference array over the concatenated contigs
    dev = torch.device("cuda", cluster._context().device)
    p = torch.from_numpy(pairs).to(dev).long()
    nb = torch.from_numpy(asm.lengths // res + 1).to(dev)
    off = torch.cumsum(nb, 0) - nb
    m = (p[:, 0] == p[:, 2]) & (p[:, 0] >= 0) & (p[:, 0] < n)
    c, lo, hi = p[m, 0], torch.minimum(p[m, 1], p[m, 3]), torch.maximum(p[m, 1], p[m, 3])
    s = torch.clamp(lo // res, max=nb[c])
    e = torch.clamp(hi // res + 1, max=nb[c])
    d = torch.zeros(int(nb.sum()) + 1, dtype=torch.int64, device=dev)
    d.index_add_(0, off[c] + s, (s < e).long())
    d.index_add_(0, off[c] + e, -(s < e).long())
    want = torch.cumsum(d[:-1], 0).to(torch.int32).cpu().numpy()
    got = np.concatenate([cov[f] for f in range(n)])
    assert np.array_equal(got, want)
    del p, d
    # breakpoints of round 1 against the oracle on the same coverage
    corr.round(0.2, 0.1, 5000, True)
    frag, bins, bcov = corr.breaks()
    want_b = []
    for f in range(n):
        for pos, cv in orc.detect(cov[f], int(asm.lengths[f]), res):
            want_b.append((f, pos // res, cv))
    assert list(zip(frag.tolist(), bins.tolist(), bcov.tolist())) == want_b
    # the second half of the planted junctions are zero-coverage gaps of +- 1000 bp (synth.chimera_case): each must have
    # coverage 0 at its bin, and every one the oracle breaks there must be broken by the device at the same bin
    zero = junctions[len(junctions) // 2:]
    assert len(zero) == 60 and all(cov[cid][pos // res] == 0 for cid, pos in zero)
    dev_b = set(zip(frag.tolist(), bins.tolist()))
    zb = [(f, b) for f, b, cv in want_b if cv == 0]
    hit = [(cid, pos) for cid, pos in zero if any(f == cid and abs(b * res - pos) <= 1000 for f, b in zb)]
    assert len(hit) >= 54, len(hit)
    for cid, pos in hit:
        mine = [(f, b) for f, b in zb if f == cid and abs(b * res - pos) <= 1000]
        assert all(x in dev_b for x in mine), (cid, pos)
    print("planted junctions: {} ({} zero-coverage, {} of them broken in the gap), contigs broken: {}, zero breakpoints: {}".format(
        len(junctions), len(zero), len(hit), len(set(frag.tolist())), len(zb)))
    # remap against torch.searchsorted on a layout that breaks every contig at its breakpoints
    base, starts, ids = [0], [], []
    nid = 0
    by = {}
    for f, b, _ in want_b:
        by.setdefault(f, []).append(b * res)
    for f in range(n):
        for st in [0] + by.get(f, []):
            starts.append(st)
            ids.append(nid)
            nid += 1
        base.append(len(starts))
    layout = (np.array(base, np.int32), np.array(starts, np.int64), np.array(ids, np.int32))
    corr.set_layout(*layout)
    sub = pairs[:5_000_000]
    got = corr.remap(sub)
    src = torch.repeat_interleave(torch.arange(n, device=dev), torch.from_numpy(np.diff(layout[0])).to(dev).long())
    key = src * (1 << 33) + torch.from_numpy(layout[1]).to(dev)
    q = torch.from_numpy(sub).to(dev).long()
    out = q.clone()
    for k in (0, 2):
        j = torch.searchsorted(key, q[:, k] * (1 << 33) + q[:, k + 1], right=True) - 1
        out[:, k] = torch.from_numpy(layout[2]).to(dev).long()[j]
        out[:, k + 1] = q[:, k + 1] - torch.from_numpy(layout[1]).to(dev)[j]
    assert np.array_equal(got, out.to(torch.int32).cpu().numpy())
    corr.close()
