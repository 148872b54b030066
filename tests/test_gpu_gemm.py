"""GPU parity of the tensor-core pre-expansion (hh_mcl_create_ex, HH_PREEXP_DENSE; csrc/hh_gemm.cu) against
  * the exact (fp64) product of the fp32 matrix M0 the reference multiplies (HapHiC_cluster.py:2144-2149),
  * the reference's own golden M1 / iterates / iteration counts / clusters (tests/golden/mcl_*.npz),
  * the Gustavson engine of this library,
through the C ABI.

Tolerance: M1 within 2e-6 relative of the exact product on every stored entry and an identical non-zero pattern.  That is
the error the reference's own fp32 ascending-k SpGEMM has against the exact product (measured 0.9e-6 .. 1.7e-6 on the same
inputs), so both engines sit inside one fp32 rounding band around the same real-number result."""

import numpy as np
import pytest
import scipy.sparse as sp

from tests.util import csc_from, load_golden
from tests.test_gpu_mcl import compare_sparse, labels

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from haphic_b200._lib import Context
    c = Context(0)
    yield c
    c.close()


def random_links(n, density, maxc, seed, weights=False):
    rng = np.random.default_rng(seed)
    m = int(n * n * density / 2)
    i = rng.integers(0, n, m)
    j = rng.integers(0, n, m)
    ok = i != j
    i, j = i[ok], j[ok]
    if weights:
        v = (rng.random(len(i)) * maxc + 0.01).astype(np.float32)
    else:
        v = np.minimum(rng.geometric(0.4, len(i)), maxc).astype(np.float32)
        big = rng.random(len(i)) < 0.01
        v[big] = rng.integers(1, maxc + 1, int(big.sum())).astype(np.float32)
    a = sp.coo_matrix((v, (i, j)), shape=(n, n)).tocsr()
    a.sum_duplicates()
    a = sp.triu(a, 1)
    a = a + a.T
    if not weights:
        a.data = np.minimum(a.data, maxc)
    a = sp.csc_matrix(a + sp.identity(n, dtype=np.float32, format="csc"), dtype=np.float32)
    a.sort_indices()
    return a


def exact_m1(link):
    d = link.toarray().astype(np.float64)
    m0 = (d / d.sum(axis=0)).astype(np.float32).astype(np.float64)
    return m0 @ m0


# the operand encodings of csrc/hh_gemm.cu: (passes for integer counts, clip threshold)
ENCODINGS = {"f16": (2, 2048), "bf16": (3, 256)}


@pytest.fixture(params=sorted(ENCODINGS))
def encoding(request, monkeypatch):
    monkeypatch.setenv("HH_GEMM_FMT", request.param)
    return request.param


@pytest.mark.parametrize("n,density,maxc,weights,planes", [
    (1000, 0.3, 200, False, 1),      # small counts: one exact plane of counts
    (777, 0.5, 5000, False, 1),      # counts above the clip threshold: clipped GEMM + sparse correction; ragged tile edge
    (300, 0.5, 3, True, 3),          # float weights (--normalize_by_nlinks, allele scaling): three bf16 planes, six passes
    (100, 0.9, 40, False, 1),        # smaller than one tile
    (2600, 0.2, 300, False, 1),      # several tiles in both directions, mirror images
])
def test_dense_preexpansion_matches_exact_product(ctx, encoding, n, density, maxc, weights, planes):
    from haphic_b200.links import LinkMatrix
    from haphic_b200.mcl import Mcl
    link = random_links(n, density, maxc, seed=n, weights=weights)
    mat = LinkMatrix.from_csc(ctx, link)
    mc = Mcl(mat, preexp="dense")
    assert mc.preexp["mode"] == "dense" and mc.preexp["a_planes"] == planes
    passes, clip = ENCODINGS[encoding]
    assert mc.preexp["passes"] == (6 if weights else passes)
    assert (mc.preexp["clip_ms"] > 0) == ((not weights) and maxc > clip)
    m1 = mc.m1().astype(np.float64)
    exact = exact_m1(link)
    nz = exact != 0
    assert np.array_equal(m1 != 0, nz)
    rel = np.abs(m1[nz] - exact[nz]) / exact[nz]
    assert rel.max() <= 2e-6, rel.max()
    # the Gustavson engine on the same input: the two engines agree to twice that band
    ms = Mcl(mat, preexp="sparse")
    assert ms.preexp["mode"] == "sparse"
    m1s = ms.m1().astype(np.float64)
    assert np.array_equal(m1s != 0, nz)
    assert (np.abs(m1s[nz] - m1[nz]) / exact[nz]).max() <= 4e-6
    ms.close()
    mc.close()
    mat.close()


def test_dense_heavy_columns(ctx, encoding):
    """column sums far above 2^14: the scaled count plane of the f16 encoding is made of f16 subnormals, which must
    multiply exactly"""
    from haphic_b200.links import LinkMatrix
    from haphic_b200.mcl import Mcl
    rng = np.random.default_rng(77)
    n = 1200
    d = np.triu(rng.integers(0, 2001, (n, n)) * (rng.random((n, n)) < 0.7), 1)
    d = (d + d.T).astype(np.float32)
    np.fill_diagonal(d, 1.0)
    link = sp.csc_matrix(d)
    link.sort_indices()
    assert d.sum(axis=0).min() > 3e5
    mat = LinkMatrix.from_csc(ctx, link)
    mc = Mcl(mat, preexp="dense")
    m1 = mc.m1().astype(np.float64)
    exact = exact_m1(link)
    nz = exact != 0
    assert np.array_equal(m1 != 0, nz)
    rel = np.abs(m1[nz] - exact[nz]) / exact[nz]
    # ~840 terms of similar size per entry: the fp32 accumulation alone wanders ~sqrt(840) * 2^-24 = 1.7e-6 (SciPy's own fp32
    # product is 3e-6 off on this input); flushed subnormals would show up as errors of order 1
    assert rel.max() <= 4e-6, rel.max()
    mc.close()
    mat.close()


@pytest.mark.parametrize("chunk", ["1", "2", "4"])
def test_dense_variants(ctx, monkeypatch, chunk):
    """other drain periods give the same result within the band"""
    from haphic_b200.links import LinkMatrix
    from haphic_b200.mcl import Mcl
    monkeypatch.setenv("HH_GEMM_CHUNK", chunk)
    link = random_links(900, 0.4, 250, seed=3)
    mat = LinkMatrix.from_csc(ctx, link)
    mc = Mcl(mat, preexp="dense")
    assert mc.preexp["cta_group"] == 1 and mc.preexp["chunk_kb"] == int(chunk)
    m1 = mc.m1().astype(np.float64)
    exact = exact_m1(link)
    nz = exact != 0
    assert np.array_equal(m1 != 0, nz)
    assert (np.abs(m1[nz] - exact[nz]) / exact[nz]).max() <= 2e-6
    mc.close()
    mat.close()


def test_dense_k_chunks(ctx, monkeypatch):
    """the K range cut into several launches (what 150k contigs need: operand planes of one chunk at a time, the epilogue
    adds to M1): same accuracy, and column shards stay bit-identical to the whole run with the same cut"""
    from haphic_b200.links import LinkMatrix
    from haphic_b200.mcl import Mcl
    link = random_links(1100, 0.4, 3000, seed=21)
    mat = LinkMatrix.from_csc(ctx, link)
    exact = exact_m1(link)
    nz = exact != 0
    monkeypatch.setenv("HH_GEMM_KCHUNKS", "3")
    mc = Mcl(mat, preexp="dense")
    assert mc.preexp["k_chunks"] == 3
    whole = mc.m1()
    m1 = whole.astype(np.float64)
    assert np.array_equal(m1 != 0, nz)
    assert (np.abs(m1[nz] - exact[nz]) / exact[nz]).max() <= 2e-6
    part = Mcl(mat, col_lo=300, col_hi=777, preexp="dense")
    assert np.array_equal(part.m1(), whole[:, 300:777])
    part.close()
    mc.close()
    monkeypatch.setenv("HH_GEMM_KCHUNKS", "1")
    one = Mcl(mat, preexp="dense")
    assert one.preexp["k_chunks"] == 1
    assert np.allclose(one.m1(), whole, rtol=1e-6, atol=0)
    one.close()
    mat.close()


def test_dense_column_shards_equal_single(ctx):
    """a column shard computes every element in the same tile and orientation as the single-GPU run: bit-identical"""
    from haphic_b200.links import LinkMatrix
    from haphic_b200.mcl import Mcl
    link = random_links(1500, 0.3, 900, seed=9)
    mat = LinkMatrix.from_csc(ctx, link)
    full = Mcl(mat, preexp="dense")
    whole = full.m1()
    for lo, hi in [(0, 700), (700, 1500), (255, 258)]:
        part = Mcl(mat, col_lo=lo, col_hi=hi, preexp="dense")
        assert np.array_equal(part.m1(), whole[:, lo:hi]), (lo, hi)
        part.close()
    full.close()
    mat.close()


@pytest.mark.parametrize("tag", ["links_a", "block200", "block600"])
def test_dense_engine_reproduces_reference_goldens(ctx, tag):
    """the whole mcl() of the reference on top of the tensor-core M1: per-iteration matrices, iteration counts,
    convergence flags and clusters of the golden fixtures (made by the unmodified HapHiC_cluster.py)"""
    from haphic_b200.links import LinkMatrix
    from haphic_b200.mcl import Mcl, interpret_result
    g = load_golden("mcl_{}.npz".format(tag))
    n = len(g["link_indptr"]) - 1
    link = csc_from(g, "link", n)
    mat = LinkMatrix.from_csc(ctx, link)
    mc = Mcl(mat, expansion=int(g["expansion"]), preexp="dense")
    assert mc.preexp["mode"] == "dense"
    m1 = mc.m1()
    assert np.array_equal(m1 != 0, g["m1_dense"] != 0)
    assert np.allclose(m1, g["m1_dense"], rtol=3e-6, atol=0)      # golden = SciPy fp32 product, itself ~1e-6 off exact
    pruning = float(g["pruning"])
    for r in g["inflations"].tolist():
        key = "r{}".format(str(r).replace(".", "p"))
        k = 1
        while key + "_iter{}_indptr".format(k) in g.files:
            st = mc.run(r, max_iter=k, pruning=pruning)
            assert st["rounds"] == k
            rtol = 3e-6 * sum(r ** t for t in range(k))
            compare_sparse(mc.result(), csc_from(g, key + "_iter{}".format(k), n), rtol, (tag, key, k), max_pattern_diff=2,
                           floor=2 * pruning)
            k += 1
        st = mc.run(r, max_iter=200, pruning=pruning)
        assert st["rounds"] == int(g[key + "_niter"]), (key, st["rounds"], int(g[key + "_niter"]))
        assert st["converged"] == bool(g[key + "_converged"])
        clusters = interpret_result(mc.result())
        assert (clusters is not None) == bool(g[key + "_clusters_valid"])
        if clusters is not None:
            assert np.array_equal(labels(clusters, n), g[key + "_labels"])
    mc.close()
    mat.close()


def test_auto_selects_dense_for_dense_matrices(ctx):
    from haphic_b200.links import LinkMatrix
    from haphic_b200.mcl import Mcl
    link = random_links(3000, 1.5, 100, seed=4)        # ~1600 entries per column: 3000 * 1600^2 products vs 3 * 3000^3 / 2 flops
    mat = LinkMatrix.from_csc(ctx, link)
    mc = Mcl(mat)
    assert mc.preexp["mode"] == "dense"
    mc.close()
    sparse_link = random_links(3000, 0.02, 100, seed=5)
    mat2 = LinkMatrix.from_csc(ctx, sparse_link)
    mc2 = Mcl(mat2)
    assert mc2.preexp["mode"] == "sparse"
    mc2.close()
    mat2.close()
    mat.close()
