"""Host tests of the blocked Markov-clustering sweep (haphic_b200.mcl): the column-block planner, and the orchestration of
blocked_sweep driven by a CPU engine with the Mcl step interface, against the same engine owning every column."""

import itertools

import pytest

from haphic_b200.mcl import GEMM_TILE, blocked_sweep, plan_column_blocks
from tests.test_dist_gloo import OracleShard
from tests.util import planted_blocks


def linear_footprint(per_col, fixed):
    return lambda w: (per_col * w, fixed)


def check_plan(blocks, n, fp, budget, tile=GEMM_TILE):
    assert blocks[0][0] == 0 and blocks[-1][1] == n
    assert all(a[1] == b[0] for a, b in zip(blocks, blocks[1:]))           # contiguous
    assert all(lo < hi for lo, hi in blocks)
    assert all(hi % tile == 0 for _lo, hi in blocks[:-1])                   # aligned except the end
    assert all(sum(fp(hi - lo)) <= budget for lo, hi in blocks)


def fewest_blocks(n, fp, budget, tile=GEMM_TILE):
    """Brute force: the least number of blocks any aligned cover within the budget needs."""
    cuts = list(range(tile, n, tile))
    for k in range(1, n // tile + 2):
        for inner in itertools.combinations(cuts, k - 1):
            b = [0, *inner, n]
            if all(sum(fp(hi - lo)) <= budget for lo, hi in zip(b, b[1:])):
                return k
    raise AssertionError("no cover")


@pytest.mark.parametrize("n", [100, 128, 1000, 1025, 1300, 2000])
@pytest.mark.parametrize("per_col,fixed", [(4, 1000), (40, 0), (12, 5000)])
def test_plan_minimal_and_within_budget(n, per_col, fixed):
    fp = linear_footprint(per_col, fixed)
    for budget in sorted({fixed + per_col * w for w in (n, n - 1, 700, 520, 513, 300, 256, 200, 130, 128) if min(GEMM_TILE, n) <= w <= n}):
        blocks = plan_column_blocks(n, fp, budget)
        check_plan(blocks, n, fp, budget)
        assert len(blocks) == fewest_blocks(n, fp, budget), (n, budget, blocks)
    assert plan_column_blocks(n, fp, fixed + per_col * n) == [(0, n)]


def test_plan_narrow_last_block():
    # 2 x 640 aligned columns and the 40 left over: the budget holds 640 columns and not one more
    fp = linear_footprint(100, 10_000)
    blocks = plan_column_blocks(1320, fp, 10_000 + 100 * 640)
    assert blocks == [(0, 640), (640, 1280), (1280, 1320)]
    # a little more room: the last block absorbs the rest
    assert plan_column_blocks(1320, fp, 10_000 + 100 * 680) == [(0, 640), (640, 1320)]


def test_plan_error_names_both_sizes():
    fp = linear_footprint(1000, 50_000)
    with pytest.raises(MemoryError) as e:
        plan_column_blocks(10_000, fp, 50_000 + 1000 * 127)
    assert "128000" in str(e.value) and "50000" in str(e.value)
    with pytest.raises(MemoryError):
        plan_column_blocks(100, fp, 50_000 + 1000 * 99)       # fewer columns than a tile, and they do not fit


class HostEngine(OracleShard):
    """The oracle's column-block engine behind the constructor and close() of haphic_b200.mcl.Mcl."""
    log = []

    def __init__(self, matrix, expansion, lo, hi, preexp="auto"):
        assert expansion == 2 and preexp == "sparse"
        super().__init__(matrix.link, lo, hi)
        self.closed = False
        HostEngine.log.append(("create", lo, hi))

    def close(self):
        if not self.closed:
            HostEngine.log.append(("close",) + self.own)
        self.closed = True


class HostMatrix:
    def __init__(self, link):
        self.link = link
        self.n = link.shape[0]


def resident_run(link, r, max_iter, pruning):
    eng = OracleShard(link, 0, link.shape[0])
    eng.begin(r, pruning)
    it_nnz, rounds, conv = [], 0, False
    for it in range(max_iter):
        nnz, _prod, delta = eng.step(it)
        eng.commit()
        it_nnz.append(nnz)
        rounds = it + 1
        if it > 1 and delta <= 1e-8:
            conv = True
            break
    return eng.cur, rounds, conv, it_nnz


@pytest.mark.parametrize("blocks", [[(0, 128), (128, 180)], [(0, 64), (64, 128), (128, 180)], [(0, 180)]])
def test_blocked_sweep_equals_resident(blocks):
    from oracle import haphic_oracle as orc
    link, _ = planted_blocks(6, 30, seed=3, noise=0.5)
    n = link.shape[0]
    assert n == 180
    infl = [1.6, 2.0, 3.0]
    m1 = orc.expand(orc.col_normalize_l1(link), 2)
    HostEngine.log = []
    got = list(blocked_sweep(HostMatrix(link), 2, infl, 100, 1e-4, "sparse", blocks, engine_cls=HostEngine))
    assert [r for r, _st, _e in got] == infl                                    # sweep order
    # phase A builds the blocks one after the other and closes each before the next; the last engine runs phase B
    want_log = []
    for lo, hi in blocks[:-1]:
        want_log += [("create", lo, hi), ("close", lo, hi)]
    assert HostEngine.log == want_log + [("create",) + blocks[-1], ("close",) + blocks[-1]]
    for (r, st, _eng), (fin, rounds, conv, it_nnz) in zip(got, [resident_run(link, r, 100, 1e-4) for r in infl]):
        assert (st["rounds"], st["converged"]) == (rounds, conv)
        assert st["iter_nnz"].tolist() == it_nnz and st["nnz"] == it_nnz[-1]
        assert len(st["iter_delta"]) == len(st["iter_ms"]) == len(st["iter_products"]) == rounds
        assert st["bytes"] == 4 * n * n + 8 * it_nnz[0] + sum(16 * a + 8 * b + 12 * (n + 1) for a, b in zip(it_nnz, it_nnz[1:]))
        _want, w_rounds, w_conv = orc.mcl(m1, 2, r, 100, 1e-4)
        assert (rounds, conv) == (w_rounds, w_conv)
    # the result each yield hands out is that inflation's (read while the generator is suspended)
    HostEngine.log = []
    for r, _st, eng in blocked_sweep(HostMatrix(link), 2, infl, 100, 1e-4, "sparse", blocks, engine_cls=HostEngine):
        fin = resident_run(link, r, 100, 1e-4)[0]
        assert (eng.cur != fin).nnz == 0 and eng.cur.shape == fin.shape
