"""GPU tests of the blocked Markov-clustering sweep (haphic_b200.mcl.blocked_sweep): the pre-expanded matrix M1 built and
consumed one column block at a time must give the bytes the resident engine gives -- result CSC, rounds, convergence and
the per-iteration entry counts -- for both pre-expansion engines, uneven blocks, --expansion 3, the benchmark's matrix, and
the whole `haphic cluster` run."""

import os

import numpy as np
import pytest

from tests.test_gpu_run import DRIVER, REPO
from tests.util import load_golden

pytestmark = pytest.mark.gpu
INFLATIONS = (1.5, 2.0, 3.0)


def link_matrix(ctx, nchr, n_contigs, mean_len, n_pairs, seed):
    from haphic_b200 import synth
    from haphic_b200.links import LinkTable, name_rank
    asm = synth.make_assembly(nchr, n_contigs, mean_len, seed=seed)
    rank = name_rank(asm.names)
    in_nx = np.ones(asm.n, np.uint8)
    rec = synth.make_pairs_range(asm, 0, n_pairs, seed=seed + 1, device="cuda")
    tab = LinkTable(ctx, asm.lengths, rank, in_nx, 500000, capacity_hint=int(0.6 * min(n_pairs, asm.n * (asm.n - 1) // 2)))
    tab.add(rec, asynchronous=True)
    tab.finish()
    del rec
    keep = np.ones(asm.n, np.uint8)
    index, n_linked = tab.linked_index(keep)
    tail = np.nonzero(index < 0)[0].astype(np.int32)
    mat = tab.to_matrix(keep, tail)
    tab.close()
    ctg_of = np.empty(mat.n, np.int64)                   # matrix index -> contig id
    ctg_of[index[index >= 0]] = np.nonzero(index >= 0)[0]
    ctg_of[n_linked + np.arange(len(tail))] = tail
    return asm, mat, ctg_of


def budget_for(mat, expansion, mode, width):
    """A byte budget that holds exactly `width` columns of M1 beside the fixed footprint."""
    from haphic_b200.mcl import footprint
    m1, fixed = footprint(mat, expansion, width, mode)
    return m1 + fixed


def plan(mat, expansion, mode, width):
    from haphic_b200.mcl import footprint, plan_column_blocks
    return plan_column_blocks(mat.n, lambda w: footprint(mat, expansion, w, mode), budget_for(mat, expansion, mode, width))


def resident(mat, expansion, mode, inflations):
    from haphic_b200.mcl import Mcl
    eng = Mcl(mat, expansion, preexp=mode)
    assert eng.preexp["mode"] == mode or expansion > 2
    out = []
    for r in inflations:
        st = eng.run(r, 200, 1e-4)
        out.append((st, eng.result()))
    eng.close()
    return out


def assert_blocked_equals(mat, expansion, mode, inflations, blocks, want):
    from haphic_b200.mcl import blocked_sweep
    got = list(blocked_sweep(mat, expansion, inflations, 200, 1e-4, mode, blocks))
    assert [r for r, _st, _e in got] == list(inflations)
    for (r, st, _e), (wst, wfin) in zip(got, want):
        assert (st["rounds"], st["converged"]) == (wst["rounds"], wst["converged"]), r
        assert st["iter_nnz"].tolist() == wst["iter_nnz"].tolist(), r
        assert st["nnz"] == wst["nnz"] and st["bytes"] == wst["bytes"], r
    # the results, fetched while each inflation's engine is current
    for (r, _st, eng), (_wst, wfin) in zip(blocked_sweep(mat, expansion, inflations, 200, 1e-4, mode, blocks), want):
        fin = eng.result()
        assert np.array_equal(fin.indptr, wfin.indptr), r
        assert fin.indices.tobytes() == wfin.indices.tobytes(), r
        assert fin.data.tobytes() == wfin.data.tobytes(), r


@pytest.fixture(scope="module")
def c2_shape():
    from haphic_b200._lib import Context
    ctx = Context(0)
    asm, mat, _ctg = link_matrix(ctx, 16, 10000, 30000, 10_000_000, 12345)
    yield asm, mat
    mat.close()
    ctx.close()


@pytest.mark.parametrize("mode", ["dense", "sparse"])
def test_blocked_sweep_10k_matches_resident(c2_shape, mode):
    _asm, mat = c2_shape
    n = mat.n
    assert n == 10000
    want = resident(mat, 2, mode, INFLATIONS)
    two = plan(mat, 2, mode, 5120)
    assert two == [(0, 5120), (5120, n)]
    three = plan(mat, 2, mode, 4992)
    assert three == [(0, 4992), (4992, 9984), (9984, n)]            # the last block narrower than one GEMM tile
    for blocks in (two, three):
        assert_blocked_equals(mat, 2, mode, INFLATIONS, blocks, want)


def test_blocked_sweep_expansion3_matches_resident():
    from haphic_b200._lib import Context
    with Context(0) as ctx:
        _asm, mat, _ctg = link_matrix(ctx, 6, 2000, 30000, 2_000_000, 777)
        blocks = plan(mat, 3, "sparse", 768)
        assert blocks == [(0, 768), (768, 1536), (1536, mat.n)]
        want = resident(mat, 3, "sparse", (1.5, 2.0))
        assert_blocked_equals(mat, 3, "sparse", (1.5, 2.0), blocks, want)
        mat.close()


def test_blocked_sweep_c3_four_blocks_matches_resident():
    """The benchmark's matrix (50k contigs / 200M pairs), the engine resolved by auto, four column blocks."""
    from haphic_b200._lib import Context
    from haphic_b200.mcl import resolve_preexp
    with Context(0) as ctx:
        _asm, mat, _ctg = link_matrix(ctx, 24, 50000, 20000, 200_000_000, 12345)
        mode = resolve_preexp(mat, 2, "auto")
        blocks = plan(mat, 2, mode, 12544)
        assert len(blocks) == 4
        infl = (2.0, 3.0)
        want = resident(mat, 2, mode, infl)
        assert_blocked_equals(mat, 2, mode, infl, blocks, want)
        mat.close()


FORCE_BLOCKS = r"""
from haphic_b200 import mcl as _mcl
_plan = _mcl.plan_column_blocks
def _two_or_more(n, fp, budget, tile=_mcl.GEMM_TILE):
    half = -(-n // 2)
    blocks = _plan(n, fp, sum(fp(-(-half // tile) * tile)))
    assert len(blocks) >= 2, blocks
    with open("column_blocks.json", "w") as f:
        json.dump(blocks, f)
    return blocks
_mcl.plan_column_blocks = _two_or_more
"""


def test_cluster_run_with_blocks_matches_reference_files(tmp_path):
    import json
    import subprocess
    import sys
    g = load_golden("run_c1.npz")
    nchr, n_contigs, mean_len, n_pairs = g["shape"].tolist()
    extra = []
    for k, v in json.loads(str(g["argkw"])).items():
        extra += ["--" + k, str(v)]
    code = DRIVER.format(repo=REPO, nchr=nchr, n_contigs=n_contigs, mean_len=mean_len, n_pairs=n_pairs, seed=int(g["seed"]),
                         bam=False, extra=extra, homolog=None)
    code = code.replace("cluster.run(args", FORCE_BLOCKS + "cluster.run(args")
    env = dict(os.environ, PYTHONHASHSEED="0")
    r = subprocess.run([sys.executable, "-c", code], cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    with open(tmp_path / "column_blocks.json") as f:
        assert len(json.load(f)) >= 2
    want = json.loads(str(g["files_json"]))
    got = {}
    for root, _d, files in os.walk(tmp_path):
        for fn in files:
            p = os.path.relpath(os.path.join(root, fn), tmp_path)
            if p.startswith("inflation_") and p.endswith(".txt"):
                with open(os.path.join(root, fn)) as f:
                    got[p] = f.read()
    assert sorted(got) == sorted(want)
    for p in sorted(want):
        assert got[p] == want[p], p
    with open(tmp_path / "HapHiC_cluster.log") as f:
        log = f.read()
    assert [ln.split("] ", 1)[1] for ln in log.splitlines() if "[mcl]" in ln] == g["mcl_lines"].tolist()
    assert [ln.split("] ", 1)[1] for ln in log.splitlines() if "[recommend_inflation]" in ln] == g["recommend_lines"].tolist()


def test_c5_shape_on_one_gpu():
    """150,000 contigs (32 chromosomes, 300M pairs): the whole M1 (90 GB) exceeds the device, the sweep runs in blocks."""
    from haphic_b200._lib import Context
    from haphic_b200.cluster import _mcl_budget
    from haphic_b200.mcl import blocked_sweep, footprint, interpret_result, plan_column_blocks, resolve_preexp
    with Context(0) as ctx:
        asm, mat, ctg_of = link_matrix(ctx, 32, 150000, 20000, 300_000_000, 12345)
        n = mat.n
        mode = resolve_preexp(mat, 2, "auto")
        blocks = plan_column_blocks(n, lambda w: footprint(mat, 2, w, mode), _mcl_budget(ctx))
        assert len(blocks) >= 2
        chrom = asm.chrom[ctg_of]
        for r, st, eng in blocked_sweep(mat, 2, INFLATIONS, 200, 1e-4, mode, blocks):
            assert st["converged"], r
            fin = eng.result()
            assert abs(np.asarray(fin.sum(axis=0)).ravel() - 1.0).max() < 1e-6
            clusters = interpret_result(fin)
            assert clusters is not None and sum(len(c) for c in clusters) == n, r
            pure = sum(int(np.bincount(chrom[list(c)]).max()) for c in clusters)
            assert pure >= 0.99 * n, (r, pure)
        mat.close()
