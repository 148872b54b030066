"""Every MCL iteration engine of hh_mcl_step, step by step, against a host reference of the SAME single step computed from
the device's own previous iterate (tests/mcl_step_oracle.py).  Comparing one step at a time removes the amplification across
iterations that forces the large-n tests of test_gpu_mcl.py to compare labels only, so the bars are tight:

  sequential engines (hh_k_iter0 in the multiplicative modes, hh_k_col_win, hh_k_col_small, hh_k_col): bit-exact against
      fp32 fma in ascending i + the epilogue.  A column may differ only if its recomputation with S1 or S2 moved by one
      fp64 ulp reproduces it (a different fp64 summation order); the count is reported and expected to be 0.
  r without a multiplicative mode (powf): y = x^r within POW_ULP ulp (CUDA C++ Programming Guide, maximum ulp error of
      powf: 4), so e_y = 4 * 2^-23.
  block GEMM steps (tensor cores): the product within EPS_P = 2e-6 of the exact one (DESIGN.md section 2), so y within
      e_y = r * EPS_P.
  With a bound e_y on y: x1 = y / S1 is within 2 e_y (+ rounding), so every pattern difference must satisfy
  |x1/pruning - 1| <= 2 e_y; x2 = y / (sum of the kept y) -- S1 cancels -- is within 2 e_y + 2^-22 (three fp32 roundings).

Every case asserts through Mcl.step_info() that the engine it targets ran.  The convergence term is bit-equal to the host's
on every path.  `-s` prints the worst error of every case against its bar."""

import numpy as np
import pytest
import scipy.sparse as sp
from scipy.sparse.csgraph import connected_components

from tests import mcl_step_oracle as so

pytestmark = pytest.mark.gpu

EPS_P = 2e-6
POW_EPS = 4 * 2.0 ** -23
WINDOW_MAX = 8192          # HH_WINDOW_MAX


@pytest.fixture(scope="module")
def ctx():
    from haphic_b200._lib import Context
    c = Context(0)
    yield c
    c.close()


def make_link(sizes, seed, ring=0, band=3, strength=30.0, reach=None):
    """Symmetric link counts: a banded ring of `ring` vertices (offsets 1..band) and one block per entry of `sizes`
    (counts ~ Poisson(strength / (1 + |i - j|)), |i - j| <= reach, plus a chain that keeps the block connected), self
    loops 1, vertices shuffled so that the relabelled order differs from the original one."""
    rng = np.random.default_rng(seed)
    n = ring + int(sum(sizes))
    perm = rng.permutation(n)
    rows, cols, vals = [], [], []
    if ring:
        i = np.repeat(np.arange(ring), band)
        o = np.tile(np.arange(1, band + 1), ring)
        c = rng.poisson(strength / (1.0 + o)) + (o == 1)
        rows.append(perm[i]), cols.append(perm[(i + o) % ring]), vals.append(c)
    base = ring
    for b in sizes:
        if b > 1:
            i, j = np.triu_indices(b, 1)
            if reach is not None:
                keep = (j - i) <= reach
                i, j = i[keep], j[keep]
            c = rng.poisson(strength / (1.0 + (j - i))) + ((j - i) == 1)
            nz = c > 0
            rows.append(perm[base + i[nz]]), cols.append(perm[base + j[nz]]), vals.append(c[nz])
        base += b
    r = np.concatenate(rows) if rows else np.zeros(0, np.int64)
    c = np.concatenate(cols) if cols else np.zeros(0, np.int64)
    v = (np.concatenate(vals) if vals else np.zeros(0)).astype(np.float32)
    m = sp.coo_matrix((np.concatenate([v, v]), (np.concatenate([r, c]), np.concatenate([c, r]))), shape=(n, n)).tocsc()
    m = sp.csc_matrix(m + sp.identity(n, dtype=np.float32, format="csc"), dtype=np.float32)
    m.sum_duplicates()
    m.sort_indices()
    return m


class Report:
    def __init__(self, tag):
        self.tag = tag
        self.seq_steps = self.blk_steps = self.one_ulp = 0
        self.pow_ratio = self.blk_ratio = 0.0
        self.infos = []

    def show(self):
        print("\n[{}] sequential steps {} (one-ulp S1/S2 columns {}), block steps {} (worst x2 error / bar {:.3f}), "
              "powf worst x2 error / bar {:.3f}".format(self.tag, self.seq_steps, self.one_ulp, self.blk_steps,
                                                       self.blk_ratio, self.pow_ratio))


def _check_exact(rep, dev, X, r, pruning, mask, what):
    still, one = so.exact_bit_check(dev, X, r, pruning, mask)
    assert not still, "{}: {} columns differ from the ordered fp32 reference (first {})".format(what, len(still), still[:5])
    rep.one_ulp += len(one)


def _check_band(rep, dev, X64, r, pruning, e_y, mask, what, kind):
    res = so.band_check(dev, X64, r, pruning, e_y, mask)
    assert res["pattern_bad"] == 0, (what, res)
    assert res["max_bad"] == 0, (what, res)
    assert res["x2_err"] <= res["x2_bar"], (what, res)
    ratio = res["x2_err"] / res["x2_bar"]
    if kind == "blk":
        rep.blk_ratio = max(rep.blk_ratio, ratio)
    else:
        rep.pow_ratio = max(rep.pow_ratio, ratio)


def check_step(rep, cur, prev, info, r, pruning, win, expansion=2):
    """Iterate `cur` (host, original indices) against one step of the oracle from `prev`."""
    n = cur.shape[0]
    e_pow = 0.0 if so.special_mode(r) else POW_EPS
    seq = np.ones(n, bool)
    what = (rep.tag, info["it"])
    if info["blk"]:
        rep.blk_steps += 1
        _check_band(rep, cur, so.expand_exact(prev, win), r, pruning, r * EPS_P + e_pow, win, what, "blk")
        seq = ~win
    if not seq.any():
        return
    rep.seq_steps += 1
    if expansion == 2:
        X = so.expand_ordered(prev, seq)
    else:
        B = prev
        for _ in range(expansion - 2):
            B = so.power(prev, B)          # unpruned M^(k-1), then A . A^(k-1)
        X = so.power(prev, B)
    if e_pow == 0.0:
        _check_exact(rep, cur, X, r, pruning, seq, what)
    else:
        _check_band(rep, cur, sp.csc_matrix(X, dtype=np.float64), r, pruning, e_pow, seq, what, "pow")


def check_iter0(rep, got, m1, r, pruning, what):
    X = sp.csc_matrix(np.asarray(m1, np.float32))
    if so.special_mode(r):
        _check_exact(rep, got, X, r, pruning, None, what)
    else:
        _check_band(rep, got, sp.csc_matrix(X, dtype=np.float64), r, pruning, POW_EPS, None, what, "pow")
    rep.seq_steps += 1


def window_mask(it0):
    """Vertices whose component (pattern of the first pruned iterate, as hh_mcl_commit finds it) fits the window."""
    _nc, lab = connected_components(it0, directed=True, connection="weak")
    return np.bincount(lab)[lab] <= WINDOW_MAX


def walk(mc, r, pruning, tag, check_m1=True, max_iter=200, expansion=2, on_step=None):
    """begin / step / commit / result() to convergence, every step checked against the oracle."""
    rep = Report(tag)
    mc.begin(r, pruning)
    m1 = mc.m1() if check_m1 else None
    nnz, _p, _d = mc.step(0)
    info = mc.step_info()
    mc.commit()
    prev = so.canon(mc.result())
    assert info["iter0"] == 1 and info["it"] == 0 and nnz == prev.nnz
    rep.infos.append(info)
    if m1 is not None:
        check_iter0(rep, prev, m1, r, pruning, (tag, 0))
    win = window_mask(prev)
    for it in range(1, max_iter):
        nnz, _p, d = mc.step(it)
        info = mc.step_info()
        mc.commit()
        cur = so.canon(mc.result())
        assert info["it"] == it and info["iter0"] == 0
        assert nnz == cur.nnz, (tag, it, nnz, cur.nnz)
        assert np.float32(d) == so.delta(cur, prev), (tag, it, d, so.delta(cur, prev))
        if expansion == 2:
            assert info["n_win"] == int(win.sum()) and info["n_big"] == int((~win).sum()), (tag, it, info)
        check_step(rep, cur, prev, info, r, pruning, win, expansion)
        if on_step is not None:
            on_step(info, prev)
        rep.infos.append(info)
        prev = cur
        if it > 1 and d <= 1e-8:
            break
    rep.show()
    return rep, prev


def _mcl(ctx, link, monkeypatch, env, **kw):
    from haphic_b200.links import LinkMatrix
    from haphic_b200.mcl import Mcl
    for k, v in env.items():
        monkeypatch.setenv(k, str(v))
    mat = LinkMatrix.from_csc(ctx, link)
    return mat, Mcl(mat, **kw)


def _count(rep, **cond):
    return sum(all(i[k] == v for k, v in cond.items()) for i in rep.infos)


# ---------------------------------------------------------------------------------------------------------------------------
# 1. window components, sequential
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("r", [1.5, 2.0, 2.5, 3.0, 1.3])
def test_window_sequential_steps_bit_exact(ctx, monkeypatch, r):
    """n ~ 6000 (W = 8, row blocks of 768): components of 3..60 vertices, contiguous after the relabelling, so many of
    them straddle a row-block boundary.  hh_k_relabel_win, hh_k_col_win and hh_k_col_small, no block GEMM."""
    sizes = np.random.default_rng(11).integers(3, 61, 190).tolist()
    link = make_link(sizes, seed=12)
    mat, mc = _mcl(ctx, link, monkeypatch, {"HH_MCL_BLOCKGEMM": 0})
    rep, _ = walk(mc, r, 1e-4, "window r={}".format(r))
    assert _count(rep, blk=1) == 0
    assert _count(rep, small=0, iter0=0) >= 1, "hh_k_col_win never ran"
    assert _count(rep, small=1) >= 1, "hh_k_col_small never ran"
    assert rep.infos[0]["iter0_w"] == 8 and rep.infos[-1]["n_big"] == 0
    mc.close()
    mat.close()


# ---------------------------------------------------------------------------------------------------------------------------
# 2. overflow of the small kernel into hh_k_col
# ---------------------------------------------------------------------------------------------------------------------------
def overflow_reasons(P, cols=None):
    """The columns hh_k_col_small sends to its overflow list when it expands iterate P (columns `cols`), by the first limit
    each breaks: more than 32 entries, more than 4096 products, more than 256 result rows."""
    P = so.canon(P)
    lens = np.diff(P.indptr)
    col_of = np.repeat(np.arange(P.shape[1]), lens)
    prods = np.bincount(col_of, weights=lens[P.indices], minlength=P.shape[1])
    rows_out = np.diff(so.canon(P @ P).indptr)
    r1 = lens > 32
    r2 = ~r1 & (prods > 4096)
    r3 = ~r1 & ~r2 & (rows_out > 256)
    if cols is not None:
        r1, r2, r3 = r1 & cols, r2 & cols, r3 & cols
    return r1, r2, r3


def test_small_kernel_overflow_bit_exact(ctx, monkeypatch):
    """2000 blocks of 2-4 vertices and one banded block of 200 at r = 1.3: nnz <= 8n while the wide block's columns have
    more than 32 entries, go to the overflow list and are finished by hh_k_col, whose operands' row-block pointers were
    written by hh_k_col_win / hh_k_col_small.  MCL narrows all columns of such a block at about the same step, so only
    this first limit is met here; test_small_kernel_overflow_every_limit reaches the other two."""
    rng = np.random.default_rng(21)
    sizes = [200] + rng.integers(2, 5, 2000).tolist()
    link = make_link(sizes, seed=22, reach=60)
    mat, mc = _mcl(ctx, link, monkeypatch, {"HH_MCL_BLOCKGEMM": 0})
    reasons = np.zeros(3, np.int64)

    def tally(info, prev):
        """The overflow list must hold exactly the columns that break one of the small kernel's limits."""
        if not info["small"]:
            return
        r = overflow_reasons(prev)
        assert info["small_overflow"] == int(sum(x.sum() for x in r)), info
        reasons[:] += [x.sum() for x in r]

    rep, _ = walk(mc, 1.3, 1e-4, "small overflow", on_step=tally)
    over = [i for i in rep.infos if i["small"] and i["small_overflow"] > 0]
    assert over, "no column overflowed hh_k_col_small"
    assert all(i["col"] == 1 and i["col_cols"] == i["small_overflow"] for i in over)
    assert reasons[0] > 0
    print("overflow columns per step:", [i["small_overflow"] for i in over],
          "by limit (> 32 entries, > 4096 products, > 256 rows):", reasons.tolist())
    mc.close()
    mat.close()


def overflow_link(n_iso=3000, seed=23):
    """Vertices [0, 300 + n_iso): 300 'narrow' vertices linked to peers (count 100) and n_iso isolated ones; vertices
    [300 + n_iso, 600 + n_iso): 300 peers with self loops of 10^4.  At r = 3 iteration 0 leaves every narrow column
    with its peers and itself only: 21 entries for j < 270 (peers 0..149 for j < 100, peers 150..299 for 100 <= j < 270),
    41 for j >= 270."""
    rng = np.random.default_rng(seed)
    base = 300 + n_iso
    n = base + 300
    rows, cols = [], []
    for j in range(300):
        pool = np.arange(150) if j < 100 else (np.arange(150, 300) if j < 270 else np.arange(300))
        peers = base + rng.choice(pool, 40 if j >= 270 else 20, replace=False)
        rows.append(peers), cols.append(np.full(len(peers), j))
    r, c = np.concatenate(rows), np.concatenate(cols)
    v = np.full(len(r), 100.0, np.float32)
    diag = np.ones(n, np.float32)
    diag[base:] = 1.0e4
    m = sp.coo_matrix((np.concatenate([v, v, diag]), (np.concatenate([r, c, np.arange(n)]), np.concatenate([c, r, np.arange(n)]))),
                      shape=(n, n)).tocsc()
    return sp.csc_matrix(m, dtype=np.float32), base


def test_small_kernel_overflow_every_limit(ctx, monkeypatch):
    """A column shard steps its own columns while the peer block's columns are installed through hh_mcl_unpack (what the
    all-gather of a sharded run does): the peers' columns are wide (300 rows for peers 0..149, 150 rows for peers
    150..299, random rows of the component, positive values), the shard's own columns narrow.  Expanding them, the
    columns of narrow vertices with 41 entries break the entry limit, those pointing at 20 wide peers the product limit
    (> 4096), those pointing at 20 medium peers the result-row limit (> 256 distinct rows, 3000 products).  Every overflow
    column is finished by hh_k_col; the step is bit-exact and the overflow list holds exactly those columns."""
    import torch
    link, base = overflow_link()
    n = link.shape[0]
    mat, mc = _mcl(ctx, link, monkeypatch, {"HH_MCL_BLOCKGEMM": 0}, col_lo=0, col_hi=base)
    rng = np.random.default_rng(24)
    comp = np.concatenate([np.arange(300), np.arange(base, n)])       # the narrow vertices and the peers
    peer_cols = []
    for p in range(300):
        rows = np.sort(rng.choice(comp, 300 if p < 150 else 150, replace=False))
        vals = rng.random(len(rows)).astype(np.float32) + np.float32(0.5)
        peer_cols.append((rows, (vals / vals.sum()).astype(np.float32)))
    ln = torch.tensor([len(c[0]) for c in peer_cols], dtype=torch.int32, device="cuda")
    idx = torch.tensor(np.concatenate([c[0] for c in peer_cols]), dtype=torch.int32, device="cuda")
    val = torch.tensor(np.concatenate([c[1] for c in peer_cols]), dtype=torch.float32, device="cuda")
    own = np.zeros(n, bool)
    own[:base] = True
    r, pruning = 3.0, 1e-4
    prev = None
    rep = Report("small overflow, every limit")
    reasons = np.zeros(3, np.int64)
    mc.begin(r, pruning)
    for it in range(2):
        nnz, _p, d = mc.step(it)
        info = mc.step_info()
        if it == 0:
            mc.unpack(base, n, ln, idx, val)             # the peer block (original row indices: before the relabelling)
        mc.commit()
        cur = so.canon(mc.result())                      # after step 1 only the own columns are meaningful
        assert nnz == cur[:, :base].nnz
        if it == 0:
            assert np.diff(cur.indptr)[:300].max() == 41 and np.diff(cur.indptr)[:270].max() <= 32
        else:
            assert info["small"] == 1, info
            rs = overflow_reasons(prev, own)
            assert info["small_overflow"] == int(sum(x.sum() for x in rs)), info
            assert info["col"] == 1 and info["col_cols"] == info["small_overflow"]
            reasons += [x.sum() for x in rs]
            _check_exact(rep, cur, so.expand_ordered(prev, own), r, pruning, own, (rep.tag, it))
            assert np.float32(d) == so.delta(cur[:, :base], prev[:, :base])
            rep.seq_steps += 1
        prev = cur
    print("overflow by limit (> 32 entries, > 4096 products, > 256 rows):", reasons.tolist())
    assert (reasons > 0).all(), reasons
    rep.show()
    mc.close()
    mat.close()


# ---------------------------------------------------------------------------------------------------------------------------
# 3. components wider than the window: hh_k_col in perm space
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ring,n_total,W,smem", [(9000, 10000, 8, 1), (9000, 20000, 16, 1), (9000, 40000, 32, 1),
                                                 (9000, 60000, 32, 0)])
def test_wide_component_steps_bit_exact(ctx, monkeypatch, ring, n_total, W, smem):
    """A banded ring of 9000 vertices stays one component after iteration 0 (> HH_WINDOW_MAX): its columns are expanded by
    hh_k_col through SRC_CSC-relabelled operands, first maximum by original index.  Small blocks fill n up to W = 8 / 16 /
    32 and to the global-memory accumulator (n = 60,000), dense enough (> 8 entries per column) for the accumulator
    kernel to take the wide component's columns.  At n = 10,000 the ring's component labels need more than 64 rounds of
    hooking to converge: the relabelling used to stop there and fail with a slot overflow."""
    rng = np.random.default_rng(n_total)
    rest, sizes = n_total - ring, []
    while rest > 0:
        b = int(min(rest, rng.integers(8, 17)))
        sizes.append(b)
        rest -= b
    link = make_link(sizes, seed=n_total + 1, ring=ring, band=4)
    mat, mc = _mcl(ctx, link, monkeypatch, {"HH_MCL_BLOCKGEMM": 0})
    rep, _ = walk(mc, 2.0, 1e-4, "wide n={}".format(n_total), check_m1=n_total <= 12288)
    cols = [i for i in rep.infos if i["col"]]
    assert cols, "hh_k_col never ran"
    assert all(i["col_w"] == W and i["col_smem"] == smem for i in cols)
    assert rep.infos[-1]["n_big"] == ring
    # sparse columns: the dirty-chunk bitmap and the flat walk (the dense variants: the next test)
    assert any(i["col_track"] == 1 and i["col_flat"] == 1 for i in cols), cols[:2]
    mc.close()
    mat.close()


def test_wide_component_dense_columns_track_and_flat_off(ctx, monkeypatch):
    """Dense columns turn TRACK and FLAT off (average > 128 entries per column at W = 8): the ring's columns (hh_k_col,
    bit-exact) beside ten dense 400-blocks (block GEMM, forced, rounding band).  With the previous test, both values of
    both switches are covered."""
    link = make_link([400] * 10, seed=31, ring=8200, band=4, strength=60.0)
    assert link.shape[0] <= 12288
    mat, mc = _mcl(ctx, link, monkeypatch, {"HH_MCL_BLOCKGEMM": 2})
    rep, _ = walk(mc, 1.3, 1e-4, "track/flat", check_m1=False, max_iter=5)
    cols = [i for i in rep.infos if i["col"]]
    assert any(i["col_track"] == 0 and i["col_flat"] == 0 for i in cols), cols[:2]
    assert _count(rep, blk=1) >= 1
    mc.close()
    mat.close()


# ---------------------------------------------------------------------------------------------------------------------------
# 4. / 5. block GEMM on the tensor cores
# ---------------------------------------------------------------------------------------------------------------------------
BLK_SIZES = [1, 37, 128, 129, 300, 1000, 2100]


@pytest.mark.parametrize("r,chunk", [(1.3, None), (2.0, None), (2.0, 1), (2.0, 4)])
def test_block_gemm_f16_steps_within_band(ctx, monkeypatch, r, chunk):
    """HH_MCL_BLOCKGEMM=2 at pruning 1e-4: two f16 planes of M * 2^14, four passes.  Components 1 .. 2100: ragged tiles,
    ldk padding, several tiles per component."""
    env = {"HH_MCL_BLOCKGEMM": 2}
    if chunk is not None:
        env["HH_GEMM_CHUNK"] = chunk
    link = make_link(BLK_SIZES, seed=41)
    mat, mc = _mcl(ctx, link, monkeypatch, env)
    rep, _ = walk(mc, r, 1e-4, "blk f16 r={} chunk={}".format(r, chunk), max_iter=40)
    blk = [i for i in rep.infos if i["blk"]]
    assert len(blk) >= 2
    assert all(i["blk_f16"] == 1 and i["blk_chunk"] == (2 if chunk is None else chunk) for i in blk)
    assert all(i["blk_ldk"] == 2112 for i in blk)            # 2100 padded to 64
    mc.close()
    mat.close()


@pytest.mark.parametrize("pruning,fmt,want_f16", [(1e-5, None, 0), (6.1e-5, None, 0), (6.2e-5, None, 1), (1e-4, "bf16", 0)])
def test_block_gemm_bf16_steps_within_band(ctx, monkeypatch, pruning, fmt, want_f16):
    """Three exact bf16 planes (six passes) below pruning 6.2e-5 or with HH_GEMM_BLK_FMT=bf16; f16 at 6.2e-5."""
    env = {"HH_MCL_BLOCKGEMM": 2}
    if fmt:
        env["HH_GEMM_BLK_FMT"] = fmt
    link = make_link([37, 129, 300, 1000], seed=51)
    mat, mc = _mcl(ctx, link, monkeypatch, env)
    rep, _ = walk(mc, 2.0, pruning, "blk p={} fmt={}".format(pruning, fmt), max_iter=40)
    blk = [i for i in rep.infos if i["blk"]]
    assert len(blk) >= 2
    assert all(i["blk_f16"] == want_f16 for i in blk)
    mc.close()
    mat.close()


# ---------------------------------------------------------------------------------------------------------------------------
# 6. default dispatch
# ---------------------------------------------------------------------------------------------------------------------------
def test_default_dispatch_picks_block_gemm(ctx, monkeypatch):
    """No forcing: four dense components of 2048 (n = 8192) at r = 1.2 -- the cost model picks the block GEMM itself."""
    monkeypatch.delenv("HH_MCL_BLOCKGEMM", raising=False)
    link = make_link([2048] * 4, seed=61, strength=200.0)
    mat, mc = _mcl(ctx, link, monkeypatch, {})
    rep, _ = walk(mc, 1.2, 1e-4, "default dispatch", check_m1=False, max_iter=4)
    assert _count(rep, blk=1) >= 3
    mc.close()
    mat.close()


# ---------------------------------------------------------------------------------------------------------------------------
# 7. column shards, then replicated with the block GEMM
# ---------------------------------------------------------------------------------------------------------------------------
def test_shards_then_replicated_block_gemm(ctx, monkeypatch):
    """Two column shards exchange their blocks (pack / unpack) for three steps, then both switch to set_block(0, n) and run
    the block GEMM (phase B of dist.sharded_mcl_sweep): their iterates stay bit-identical and every step meets the band."""
    link = make_link([37, 129, 300, 1000, 5, 9], seed=71)
    n = link.shape[0]
    cut = n // 3
    mat, s0 = _mcl(ctx, link, monkeypatch, {"HH_MCL_BLOCKGEMM": 2}, col_lo=0, col_hi=cut)
    from haphic_b200.mcl import Mcl
    s1 = Mcl(mat, col_lo=cut, col_hi=n)
    r, pruning = 2.0, 1e-4
    rep = Report("shards")
    s0.begin(r, pruning)
    s1.begin(r, pruning)
    prev, win, replicated, blk_steps = None, None, False, 0
    for it in range(60):
        n0, _p0, d0 = s0.step(it)
        n1, _p1, d1 = s1.step(it)
        i0, i1 = s0.step_info(), s1.step_info()
        if not replicated:
            b0, b1 = s0.pack(n0), s1.pack(n1)
            s1.unpack(0, cut, *b0)
            s0.unpack(cut, n, *b1)
        s0.commit()
        s1.commit()
        cur = so.canon(s0.result())
        other = so.canon(s1.result())
        assert so.columns_equal(cur, other).all(), it
        if replicated:
            # the block GEMM runs on every step outside the nearly-converged branch
            assert i0["blk"] == i1["blk"] == 1 - i0["small"] and i0["small"] == i1["small"], (i0, i1)
            assert (n0, d0) == (n1, d1) and n0 == cur.nnz
            assert np.float32(d0) == so.delta(cur, prev)
            check_step(rep, cur, prev, i0, r, pruning, win)
            blk_steps += i0["blk"]
        if it == 0:
            win = window_mask(cur)
        prev = cur
        if not replicated and it >= 2:
            s0.set_block(0, n)
            s1.set_block(0, n)
            replicated = True
        elif replicated and it > 1 and max(d0, d1) <= 1e-8:
            break
    rep.show()
    assert blk_steps >= 2
    for o in (s0, s1):
        o.close()
    mat.close()


# ---------------------------------------------------------------------------------------------------------------------------
# 8. iteration 0
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_total,W", [(3000, 8), (13000, 16), (30000, 32)])
def test_iter0_bit_exact(ctx, monkeypatch, n_total, W):
    """hh_k_iter0 on a block of 256 columns (W from n), special modes bit-exact, r = 1.3 within the powf bound."""
    from haphic_b200.mcl import Mcl
    rng = np.random.default_rng(n_total)
    sizes = []
    rest = n_total
    while rest > 0:
        b = int(min(rest, rng.integers(20, 200)))
        sizes.append(b)
        rest -= b
    link = make_link(sizes, seed=n_total + 2)
    mat, mc = _mcl(ctx, link, monkeypatch, {}, col_lo=0, col_hi=256)
    rep = Report("iter0 W={}".format(W))
    m1 = mc.m1()
    for r in (1.5, 2.0, 2.5, 3.0, 1.3):
        mc.begin(r, 1e-4)
        nnz, _p, _d = mc.step(0)
        info = mc.step_info()
        assert info["iter0"] == 1 and info["iter0_w"] == W
        ln, idx, val = (t.cpu().numpy() for t in mc.pack(nnz))
        got = sp.csc_matrix((val, idx, np.concatenate([[0], np.cumsum(ln)])), shape=(n_total, 256))
        check_iter0(rep, got, m1, r, 1e-4, (rep.tag, r))
    rep.show()
    mc.close()
    if W == 8:
        # a column shard's iteration 0 == the same columns of the whole run
        whole = Mcl(mat)
        whole.begin(2.0, 1e-4)
        whole.step(0)
        whole.commit()
        full = so.canon(whole.result())[:, :256]
        sh = Mcl(mat, col_lo=0, col_hi=256)
        sh.begin(2.0, 1e-4)
        nnz, _p, _d = sh.step(0)
        ln, idx, val = (t.cpu().numpy() for t in sh.pack(nnz))
        part = sp.csc_matrix((val, idx, np.concatenate([[0], np.cumsum(ln)])), shape=(n_total, 256))
        assert so.columns_equal(part, full).all()
        whole.close()
        sh.close()
    mat.close()


@pytest.mark.parametrize("shift", [0, -1, 1])
def test_iter0_pruning_on_an_occurring_value(ctx, monkeypatch, shift):
    """The pruning threshold placed exactly on an x1 value that occurs (and on its fp32 neighbours): entries with
    x1 == pruning are kept, which tests the candidate cut xthr of hh_k_iter0."""
    link = make_link(np.random.default_rng(81).integers(20, 120, 40).tolist(), seed=82)
    mat, mc = _mcl(ctx, link, monkeypatch, {})
    m1 = sp.csc_matrix(mc.m1())
    for r in (2.0, 1.5):
        _res, im = so.epilogue(m1, r, 1e-4)
        x1 = np.sort(im["x1"])
        v = x1[np.searchsorted(x1, np.float32(3e-3))]     # an occurring x1 near 3e-3
        for _ in range(abs(shift)):
            v = np.nextafter(v, np.float32(np.inf if shift > 0 else 0))
        pruning = float(v)
        hits = int(np.count_nonzero(im["x1"] == np.float32(pruning)))
        assert shift != 0 or hits >= 1
        mc.begin(r, pruning)
        nnz, _p, _d = mc.step(0)
        mc.commit()
        got = so.canon(mc.result())
        assert nnz == got.nnz
        still, one = so.exact_bit_check(got, m1, r, pruning)
        assert not still, (r, shift, still[:5])
    mc.close()
    mat.close()


# ---------------------------------------------------------------------------------------------------------------------------
# 9. --expansion 3
# ---------------------------------------------------------------------------------------------------------------------------
def test_expansion3_steps_bit_exact(ctx, monkeypatch):
    """--expansion 3 at W = 16 (n = 13,000): no relabelling; hh_k_col computes the unpruned M^2 of the owned columns
    (raw_product), then M . M^2 with the prune epilogue and the convergence term against M."""
    rng = np.random.default_rng(91)
    sizes, rest = [], 13000
    while rest > 0:
        b = int(min(rest, rng.integers(3, 12)))
        sizes.append(b)
        rest -= b
    link = make_link(sizes, seed=92)
    mat, mc = _mcl(ctx, link, monkeypatch, {}, expansion=3)
    rep, _ = walk(mc, 2.0, 1e-4, "expansion 3", check_m1=False, expansion=3, max_iter=60)
    cols = [i for i in rep.infos if i["col"]]
    assert cols and all(i["col_w"] == 16 for i in cols)
    assert rep.seq_steps >= 2
    mc.close()
    mat.close()
