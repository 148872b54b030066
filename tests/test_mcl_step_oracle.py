"""CPU checks of the one-step MCL oracle (tests/mcl_step_oracle.py) that the GPU step tests rely on: the exact fp32 fma
against rational arithmetic, the ordered expansion against a scalar loop, the epilogue and the convergence term against
oracle/haphic_oracle.py, and expansion + epilogue against the golden iterates of the reference."""

import math
from fractions import Fraction

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import haphic_oracle as orc
from tests import mcl_step_oracle as so
from tests.util import csc_from, load_golden


def _round_f32(q: Fraction) -> np.float32:
    """Correct (nearest-even) rounding of a rational to fp32."""
    if q == 0:
        return np.float32(0)
    sign = -1 if q < 0 else 1
    q = abs(q)
    e = math.floor(math.log2(q.numerator) - math.log2(q.denominator))
    while Fraction(2) ** e > q:
        e -= 1
    while Fraction(2) ** (e + 1) <= q:
        e += 1
    e = max(e, -126)                                   # subnormal spacing below 2^-126
    ulp = Fraction(2) ** (e - 23)
    m = q / ulp
    f = math.floor(m)
    rem = m - f
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and f % 2 == 1):
        f += 1
    return np.float32(sign * float(f * ulp))


def _fma_exact(a, b, c):
    return _round_f32(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def test_fma32_random_matches_rational():
    rng = np.random.default_rng(1)
    k = 3000
    a = (rng.random(k) * 2 - 0.5).astype(np.float32) * np.float32(2.0) ** rng.integers(-30, 10, k).astype(np.float32)
    b = (rng.random(k) * 2 - 0.5).astype(np.float32) * np.float32(2.0) ** rng.integers(-30, 10, k).astype(np.float32)
    c = (rng.random(k) * 2 - 0.5).astype(np.float32) * np.float32(2.0) ** rng.integers(-40, 10, k).astype(np.float32)
    got = so.fma32(a, b, c)
    want = np.array([_fma_exact(x, y, z) for x, y, z in zip(a, b, c)], np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_fma32_halfway_cases():
    """Constructed ties and near-ties of the fp32 rounding, where a double rounding (fp64 then fp32) goes wrong."""
    one = np.float32(1.0)
    cases = []
    for m in range(1, 200):
        base = np.float32(1.0 + m * 2.0 ** -23)            # a fp32 with a known last bit
        # a * b = 2^-24 exactly (half an ulp of `base`), plus / minus a tiny amount through a second product term
        cases.append((np.float32(2.0 ** -12), np.float32(2.0 ** -12), base))
        cases.append((np.float32(2.0 ** -12), np.float32(2.0 ** -12 * (1 + 2.0 ** -23)), base))
        cases.append((np.float32(2.0 ** -12), np.float32(2.0 ** -12 * (1 - 2.0 ** -24)), base))
        cases.append((np.float32(-(2.0 ** -12)), np.float32(2.0 ** -12), base))
        # the exact sum is a tie of fp32 but its fp64 rounding is not: product bits beyond 53 decide
        x = np.float32(1 + 2.0 ** -23 * m)
        y = np.float32(1 + 2.0 ** -22)
        cases.append((x, y, np.float32(-1.0)))
        cases.append((x, y, base))
        # a * b + c just off an fp32 midpoint by less than half an fp64 ulp: the fp64 sum lands ON the midpoint and a
        # plain cast to fp32 rounds to even, the wrong way for half of these (what the round-to-odd step corrects)
        for k in range(14, 21):
            x = 2.0 ** -k
            for sign in (1.0, -1.0):
                cases.append((np.float32(2.0 ** -12 * (1 + x)), np.float32(sign * 2.0 ** -12 * (1 - x)), base))
    a, b, c = (np.array(t, np.float32) for t in zip(*cases))
    got = so.fma32(a, b, c)
    want = np.array([_fma_exact(x, y, z) for x, y, z in cases], np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    # the non-fused evaluation differs on some of them, and so does an fp64 fma rounded twice: the cases are not vacuous
    assert np.any((a * b + c).view(np.uint32) != want.view(np.uint32))
    twice = (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)
    assert np.count_nonzero(twice.view(np.uint32) != want.view(np.uint32)) >= 100
    assert so.fma32(one, one, np.float32(0)) == one


def _random_stochastic(n, density, seed):
    rng = np.random.default_rng(seed)
    a = sp.random(n, n, density=density, random_state=rng, format="csc", dtype=np.float64)
    a = a + sp.identity(n)
    return orc.col_normalize_l1(sp.csc_matrix(a, dtype=np.float32))


def test_expand_ordered_matches_scalar_loop():
    P = so.canon(_random_stochastic(40, 0.15, 3))
    n = P.shape[0]
    want = np.zeros((n, n), np.float32)
    for j in range(n):
        for p in range(P.indptr[j], P.indptr[j + 1]):
            i, b = P.indices[p], P.data[p]
            for q in range(P.indptr[i], P.indptr[i + 1]):
                r = P.indices[q]
                want[r, j] = _fma_exact(P.data[q], b, want[r, j])
    got = so.expand_ordered(P).toarray()
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert np.array_equal(so.power(P, P).toarray().view(np.uint32), want.view(np.uint32))
    mask = np.zeros(n, bool)
    mask[::3] = True
    part = so.expand_ordered(P, mask).toarray()
    assert np.array_equal(part[:, mask].view(np.uint32), want[:, mask].view(np.uint32))
    assert not part[:, ~mask].any()
    # the fp64 product agrees to fp32 rounding, also with the dense per-component path
    for dense_from in (1, 10 ** 9):
        ex = so.expand_exact(P, dense_from=dense_from).toarray()
        assert np.allclose(ex, want, rtol=1e-6, atol=0)
        assert np.array_equal(ex != 0, want != 0)


@pytest.mark.parametrize("tag", ["block200", "block600", "links_a"])
def test_epilogue_matches_oracle_inflate_prune(tag):
    """Iteration 0 of every inflation of the golden fixtures: the step epilogue == oracle.prune(oracle.inflate(M1))."""
    g = load_golden("mcl_{}.npz".format(tag))
    m1 = sp.csc_matrix(g["m1_dense"].astype(np.float32))
    pruning = float(g["pruning"])
    for r in list(g["inflations"].tolist()) + [1.5, 2.5, 3.0]:
        got, im = so.epilogue(m1, r, pruning)
        want = so.canon(orc.prune(orc.inflate(m1, r), pruning))
        got = so.canon(got)
        assert np.array_equal(got.indptr, want.indptr) and np.array_equal(got.indices, want.indices), (tag, r)
        if so.special_mode(r) == "sq":
            # numpy's power(x, 2) is x * x: the only differences left are the summation orders (fsum vs sequential fp64)
            assert np.count_nonzero(got.data != want.data) <= 0.001 * got.nnz + 1, (tag, r)
        np.testing.assert_array_max_ulp(got.data, want.data, maxulp=4)
        assert len(im["S1"]) == m1.shape[1]


@pytest.mark.parametrize("tag", ["block200", "block600", "links_a"])
def test_exact_step_matches_golden_iterates(tag):
    """expand_exact + epilogue applied to golden iterate k-1 gives golden iterate k, within the bars of test_gpu_mcl.py."""
    from tests.test_gpu_mcl import compare_sparse
    g = load_golden("mcl_{}.npz".format(tag))
    n = len(g["link_indptr"]) - 1
    pruning = float(g["pruning"])
    checked = 0
    for r in g["inflations"].tolist():
        key = "r{}".format(str(r).replace(".", "p"))
        k = 2
        while key + "_iter{}_indptr".format(k) in g.files:
            prev = csc_from(g, key + "_iter{}".format(k - 1), n)
            X = so.expand_exact(prev)
            got, _ = so.epilogue(sp.csc_matrix(X, dtype=np.float32), r, pruning)
            compare_sparse(got, csc_from(g, key + "_iter{}".format(k), n), 2e-6 * (1 + r), (tag, key, k),
                           max_pattern_diff=2, floor=2 * pruning)
            k += 1
            checked += 1
    assert checked > 0


@pytest.mark.parametrize("tag", ["block200", "block600"])
def test_delta_matches_oracle_convergence_delta(tag):
    g = load_golden("mcl_{}.npz".format(tag))
    n = len(g["link_indptr"]) - 1
    for r in g["inflations"].tolist():
        key = "r{}".format(str(r).replace(".", "p"))
        k = 2
        while key + "_iter{}_indptr".format(k) in g.files:
            a = csc_from(g, key + "_iter{}".format(k), n)
            b = csc_from(g, key + "_iter{}".format(k - 1), n)
            assert so.delta(a, b) == np.float32(orc.convergence_delta(a, b))
            assert so.delta(b, b) == 0
            k += 1


def test_column_compare_and_band_check_detect_differences():
    P = _random_stochastic(60, 0.1, 5)
    X = so.expand_ordered(P)
    res, _ = so.epilogue(X, 2.0, 1e-4)
    assert so.exact_bit_check(res, X, 2.0, 1e-4) == ([], [])
    bad = res.copy()
    bad.data[7] = np.nextafter(bad.data[7], np.float32(1))
    still, one = so.exact_bit_check(bad, X, 2.0, 1e-4)
    assert len(still) == 1 and one == []
    ok = so.band_check(res, so.expand_exact(P), 2.0, 1e-4, e_y=2 * 2e-6)
    assert ok["pattern_bad"] == 0 and ok["max_bad"] == 0 and ok["x2_err"] <= ok["x2_bar"]
    off = res.copy()
    off.data[3] *= np.float32(1 + 1e-4)
    assert so.band_check(off, so.expand_exact(P), 2.0, 1e-4, e_y=2 * 2e-6)["x2_err"] > 1e-5
